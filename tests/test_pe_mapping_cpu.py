"""Position-encoded mapping networks (use_positional_encoding_mapping1/2 of the configs): host-side network codes,
flat layouts and the single-layer script's architecture check.  No GPU work."""
import ctypes as C
import json
import os

import pytest

from b200 import _native as N
from b200 import atlas as A
from csrc_build import ensure_built

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "all-in-one-deflicker_b200")


@pytest.fixture(scope="module", autouse=True)
def _built():
    ensure_built()


def _mapping(pe, layers=6, hidden=256, skips=()):
    return A.make_desc(3, 2, hidden, layers, pe, skips)


def test_pe_mapping_architecture_code():
    lib = N.lib()
    code = lambda d: lib.b200_mlp_tc_architecture(C.byref(d))
    for pe in (1, 4, 10):
        for layers in (4, 6):
            assert code(_mapping(pe, layers)) == 4, (pe, layers)
    assert code(_mapping(11)) == 0                       # 66 encoding columns do not fit one 64-column chunk
    assert code(_mapping(4, hidden=128)) == 0
    assert code(_mapping(4, skips=(2,))) == 0
    assert code(_mapping(4, layers=8)) == 0
    assert code(A.make_desc(3, 1, 256, 6, 4, ())) == 0   # 3-input PE network with one output but not the alpha shape
    # the existing shapes keep their codes
    assert [code(d) for d in (_mapping(0), _mapping(0, 4), A.make_desc(3, 1, 256, 8, 5, ()),
                              A.make_desc(**A.ATLAS_DESC))] == [1, 1, 3, 2]


@pytest.mark.parametrize("pe", [1, 4, 10])
def test_param_floats_for_pe_mapping(pe):
    lib = N.lib()
    m, a = _mapping(pe), A.make_desc(**A.ATLAS_DESC)
    mw, mb, mt = A.mlp_layout(m)
    _, _, at = A.mlp_layout(a)
    assert lib.b200_atlas_param_floats_for(C.byref(m)) == mt + at
    assert A.layer_dims(m)[0] == (6 * pe, 256)
    assert mw[1] == (mb[0] + 256 + 3) // 4 * 4 and mb[0] == (6 * pe * 256 + 3) // 4 * 4
    # the default mapping through the new entry point is the old count
    assert lib.b200_atlas_param_floats_for(C.byref(_mapping(0))) == lib.b200_atlas_param_floats() == 681088


def test_step_entry_points_refuse_other_mappings():
    lib = N.lib()
    cfg = N.AtlasConfig(1000, 1, N.PREC_TC, 768, 0.8, 1, 100, 5000, 1000, 1, 5, 500)
    for bad in (_mapping(4, layers=4), _mapping(11), _mapping(0, layers=4), A.make_desc(3, 2, 256, 6, 4, (), False)):
        assert lib.b200_atlas_param_floats_for(C.byref(bad)) == -1
        assert lib.b200_atlas_workspace_bytes_for(C.byref(cfg), C.byref(bad)) == -1
        assert b"6-layer mapping" in lib.b200_last_error()
        assert lib.b200_render_workspace_bytes_for(C.byref(bad), 1000) == -1
    # a PE mapping needs the encoding images on top of the default mapping's buffers, in both precisions
    for prec in (N.PREC_FP32, N.PREC_TC):
        cfg.precision = prec
        base = lib.b200_atlas_workspace_bytes(C.byref(cfg))
        assert lib.b200_atlas_workspace_bytes_for(C.byref(cfg), C.byref(_mapping(0))) == base
        assert lib.b200_atlas_workspace_bytes_for(C.byref(cfg), C.byref(_mapping(4))) > base
    assert lib.b200_render_workspace_bytes_for(C.byref(_mapping(0)), 1000) == lib.b200_render_workspace_bytes(1000)
    assert lib.b200_render_workspace_bytes_for(C.byref(_mapping(10)), 1000) >= lib.b200_render_workspace_bytes(1000)


def test_check_architecture_accepts_the_pe_mapping():
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    for pe in (1, 4, 10):
        A.check_architecture(dict(cfg, use_positional_encoding_mapping1=True, number_of_positional_encoding_mapping1=pe))
        assert A.mapping_pe_freqs(dict(cfg, use_positional_encoding_mapping1=True,
                                       number_of_positional_encoding_mapping1=pe)) == pe
    assert A.mapping_pe_freqs(cfg) == 0 and A.mapping_pe_freqs(None) == 0
    for pe in (0, 11, 4.0, None):
        with pytest.raises(N.B200Error):
            A.check_architecture(dict(cfg, use_positional_encoding_mapping1=True, number_of_positional_encoding_mapping1=pe))
    # the other non-default values stay refused, with or without the encoding
    for key, val in (("number_of_layers_mapping1", 4), ("positional_encoding_num_atlas", 6), ("number_of_channels_atlas", 128)):
        for pe_on in (False, True):
            with pytest.raises(N.B200Error):
                A.check_architecture(dict(cfg, use_positional_encoding_mapping1=pe_on, **{key: val}))
