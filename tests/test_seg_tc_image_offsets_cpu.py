"""b200_seg_tc_image_offsets, host only: where each tensor-core network of a segmentation trip keeps its operand
images inside the trip's workspace (test_seg_tc_layers_gpu.py decodes them).  No device is needed: the call only
plans.  For both regimes (with / without the global rigidity term) and all four networks the images must lie inside
b200_seg_workspace_bytes, after the trip's own buffers, with [11] = the rows the trip passes the network (groups x
cap), and the four networks' image ranges must not overlap."""
import ctypes as C

import pytest

from b200 import _native as N
from b200 import seg as SG

OFFSETS, GMAX = 61, 60
MAXL = 16
TM, HID = 128, 256
CHUNK = 4 * 16384                 # bytes of one 64-wide k chunk of weight items
WS = 1 << 30                      # a 1024-aligned stand-in for the workspace address: the call does not touch it


def _trainer(batch, config=None, precision=N.PREC_TC):
    cfg = {"samples_batch": batch}
    cfg.update(config or {})
    return SG.SegTrainer(None, None, cfg, precision=precision, device="cpu")


def _offsets(cfg, net):
    out = (C.c_int64 * OFFSETS)()
    rc = N.lib().b200_seg_tc_image_offsets(C.byref(cfg), C.c_void_p(WS), net, out)
    return rc, [int(v) for v in out]


def _extent(o, desc):
    """[first byte, last byte + 1) of every image of one network, from its offset vector."""
    L, out, pe = desc.num_layers, desc.output_dim, desc.pe_freqs > 0
    k_last = HID + (2 * desc.input_dim * desc.pe_freqs if desc.skip_mask >> (L - 1) & 1 else 0)
    n_cst = (L - 1) * HID + (0 if pe else 3 * HID) + out * k_last + out
    spans = [(o[0], o[0] + max(o[12 + l] + o[12 + MAXL + l] * CHUNK for l in range(L))),
             (o[1], o[1] + max(o[12 + 2 * MAXL + l] for l in range(L)) + 4 * CHUNK),
             (o[2], o[2] + 4 * n_cst),
             (o[3], o[3] + (L - 1) * o[8]), (o[4], o[4] + (L - 1) * o[8]),
             (o[6], o[6] + 2 * o[10]), (o[7], o[7] + (L - 1) * o[11] * 32), (o[GMAX], o[GMAX] + 8)]
    if pe:
        spans.append((o[5], o[5] + 2 * o[10]))
    else:
        assert o[5] == -1
    return min(a for a, _ in spans), max(b for _, b in spans)


@pytest.mark.parametrize("batch", [1, 129, 10000])
@pytest.mark.parametrize("it", [0, 6000], ids=["with_global", "without_global"])
@pytest.mark.parametrize("pe_mappings", [False, True], ids=["plain", "pe_mappings"])
def test_images_inside_workspace_and_disjoint(it, batch, pe_mappings):
    tr = _trainer(batch, {"use_positional_encoding_mapping1": pe_mappings,
                          "use_positional_encoding_mapping2": pe_mappings})
    cfg = tr._config(it)
    assert bool(cfg.with_global) == (it == 0)
    lib = N.lib()
    nbytes = int(lib.b200_seg_workspace_bytes(C.byref(cfg)))
    trip = (C.c_int64 * N.SEG_OFFSET_FLOATS)()
    N.check(lib.b200_seg_workspace_offsets(C.byref(cfg), C.c_void_p(WS), trip), "trip offsets")
    cap = -(-batch // TM) * TM
    trip_end = trip[14] + 6 * cap * 8                       # d_xat [6][cap][2], the last buffer of the trip
    groups = {0: 9 if cfg.with_global else 7, 1: 9 if cfg.with_global else 7, 2: 5, 3: 6}
    ranges = []
    for net, which in enumerate(SG.NETS):
        rc, o = _offsets(cfg, net)
        assert rc == 0, (which, N.last_error())
        assert o[11] == groups[net] * cap, (which, o[11])
        assert o[9] == o[11] // TM * TM * HID * 2 and o[8] == 2 * o[9]
        lo, hi = _extent(o, tr.descs[which])
        assert trip_end <= lo < hi <= nbytes, (which, trip_end, lo, hi, nbytes)
        ranges.append((lo, hi, which))
    ranges.sort()
    for (_, hi, a), (lo, _, b) in zip(ranges, ranges[1:]):
        assert hi <= lo, (a, b)


def test_fp32_networks_are_refused():
    """fp32 precision has no tensor-core images at all; under B200_PREC_TC a mapping whose shape has no tensor-core
    kernels (128 channels) runs on the fp32 kernels, and only that network is refused."""
    cfg = _trainer(300, precision=N.PREC_FP32)._config(0)
    for net in range(4):
        rc, _ = _offsets(cfg, net)
        assert rc != 0 and "fp32" in N.last_error(), N.last_error()
    cfg = _trainer(300, {"number_of_channels_mapping2": 128})._config(0)
    for net in range(4):
        rc, _ = _offsets(cfg, net)
        assert (rc != 0) == (net == 1), (net, N.last_error())
    rc, _ = _offsets(cfg, 1)
    assert rc != 0 and "network 1" in N.last_error() and "fp32" in N.last_error(), N.last_error()
    rc, _ = _offsets(cfg, 4)
    assert rc != 0 and "0..3" in N.last_error()
