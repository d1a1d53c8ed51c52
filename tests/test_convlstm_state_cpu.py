"""The stateful TransformNet restatement (tests/convlstm_state_common.py) replayed against the reference fixture
(tests/golden/make_golden_convlstm_state.py),
and the host-side refusals of the ConvLSTM / packed-slice entry points.  CPU only: every refusal here happens before
any device work, so the pointers passed are never dereferenced."""
import ctypes as C
import os

import pytest
import torch

from b200 import _native as N
from convlstm_state_common import SAMPLE_STRIDE, recurrence, recurrence_inputs, transformnet_forward_state
from csrc_build import ensure_built
from nets_common import seeded_weights


def _matches(t, dg, what):
    """An output against the fixture's digest of the reference's: the sampled elements within 2e-5 (the tolerance of
    test_oracle_nets_golden.py) and the float64 sums within 2e-5 per element."""
    flat = t.reshape(-1)
    torch.testing.assert_close(flat[::SAMPLE_STRIDE], dg["sample"], atol=2e-5, rtol=0, msg=what)
    n = flat.numel()
    assert abs(float(flat.double().sum() - dg["sum"])) <= 2e-5 * n, what
    assert abs(float(flat.double().abs().sum() - dg["abs_sum"])) <= 2e-5 * n, what


def test_stateful_transformnet_restatement_replays_the_reference(golden_dir):
    """4-frame recurrence (each call fed the previous call's state) and one random-state step against the reference's
    outputs frozen by make_golden_convlstm_state.py."""
    torch.set_num_threads(1)
    fx = torch.load(os.path.join(golden_dir, "transformnet_state.pt"))
    sd = seeded_weights(fx["shapes"], fx["seed"])
    xs, x_r, state_r = recurrence_inputs(fx["input_seed"], nf=fx["nf"])
    ys, state = recurrence(sd, xs)
    for t, y in enumerate(ys):
        _matches(y, fx["ys"][t], f"frame {t} Y")
    _matches(state[0], fx["hidden"], "last hidden")
    _matches(state[1], fx["cell"], "last cell")
    y, h, c = transformnet_forward_state(sd, x_r, state_r)
    _matches(y, fx["r_y"], "random-state Y")
    _matches(h, fx["r_hidden"], "random-state hidden")
    _matches(c, fx["r_cell"], "random-state cell")
    assert float(c.abs().max()) > 6.0                     # the random state drives the cell well out of tanh's linear part


def _gates_desc(n=1, cin=256, h=16, w=24, cout=512, **kw):
    d = N.ConvDesc(n, cin, h, w, cin, 0, cout, 3, 3, 1, 1, 1, 0, 1, cout, 0, 0, 1.0, 0, 0, 0)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


FAKE = C.c_void_p(1 << 20)                                  # 256-byte aligned, never touched: refused first


@pytest.fixture(scope="module")
def lib():
    ensure_built()
    return N.lib()


@pytest.mark.parametrize("c,c_off", [(128, 132), (124, 128), (128, 136), (136, 128), (0, 0), (128, -8), (8, 256)])
def test_pack_chain_refuses_slices_it_cannot_write(lib, c, c_off):
    """b200_conv_tma_pack_chain writes 8-channel vectors: a slice that is not 8-aligned, is empty or leaves the
    consumer's input channels is refused with a message (a 256-channel consumer; [128, 256) is the hidden state's
    slice in TransformNet)."""
    rc = lib.b200_conv_tma_pack_chain(C.byref(_gates_desc()), FAKE, c, FAKE, c_off, None)
    assert rc != 0
    msg = lib.b200_last_error()
    assert b"multiple of 8" in msg and b"inside" in msg, msg


def test_pack_chain_refuses_consumers_without_a_packed_input(lib):
    strided = _gates_desc(stride=2)
    assert lib.b200_conv_tma_pack_chain(C.byref(strided), FAKE, 128, FAKE, 0, None) != 0
    assert b"pre-packed" in lib.b200_last_error()
    rc = lib.b200_conv_tma_pack_chain(C.byref(_gates_desc()), FAKE, 128, C.c_void_p((1 << 20) + 16), 128, None)
    assert rc != 0 and b"256-byte" in lib.b200_last_error()


@pytest.mark.parametrize("field,value", [("Cout", 500), ("Cout", 496), ("stride", 2), ("act", 2), ("out_scale", 0.5),
                                         ("out_c_off", 8), ("res_c_total", 512), ("upsample", 2)])
def test_convlstm_refuses_descriptors_that_are_not_a_gate_layer(lib, field, value):
    """Cout = 4C with C % 8 == 0, stride 1, no activation / scale / output slice / residual / upsampling: anything else is
    refused by both the weight-image builder and the layer, with a message."""
    d = _gates_desc(**{field: value})
    if field == "out_c_off":
        d.out_c_total = d.Cout + value
    assert lib.b200_convlstm_tma_weight_images(C.byref(d), FAKE, FAKE, None) != 0
    assert b"ConvLSTM gates" in lib.b200_last_error()
    rc = lib.b200_convlstm_tma(C.byref(d), FAKE, None, FAKE, FAKE, None, FAKE, None, FAKE, 1 << 30, None)
    assert rc != 0
    assert b"ConvLSTM gates" in lib.b200_last_error()
