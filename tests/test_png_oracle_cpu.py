"""The PNG encoder's ground on the host: the restated filter choice and file assembly (tests/png_oracle.py) equal the
installed OpenCV's level-0 PNG byte for byte, the shape-only layout b200.png.layout takes from a blank image is the
layout of any content, and b200_png_plan refuses layouts that do not add up."""
import ctypes as C

import cv2
import numpy as np
import pytest

import png_oracle as O
from b200 import _native as N
from b200 import png as P
from csrc_build import ensure_built

SHAPES = [(1, 1), (1, 2), (2, 1), (17, 5), (3, 7), (64, 100), (1, 22000), (5, 21846), (270, 1440), (333, 211)]


@pytest.fixture(scope="module", autouse=True)
def _built():
    ensure_built()


def _cv2(img):
    ok, buf = cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, 0])
    assert ok
    return buf.tobytes()


@pytest.mark.parametrize("h,w", SHAPES, ids=lambda v: str(v))
def test_restated_writer_equals_opencv(h, w):
    lay = P.layout(h, w)
    for kind in O.KINDS:
        img = O.content(kind, h, w)
        want = _cv2(img)
        assert np.array_equal(O.filter_rows(img)[0], O.idat_filters(want, h, w)), kind
        assert O.encode(img, lay) == want, kind


@pytest.mark.parametrize("h,w", [(1080, 1920), (1080, 5760)], ids=lambda v: str(v))
def test_restated_writer_equals_opencv_at_stage2_sizes(h, w):
    img = O.content("random", h, w)
    assert O.encode(img, P.layout(h, w)) == _cv2(img)


def test_tie_contents_tie():
    """The tie images do what they are for: shared minima, and Paeth picked on rows where its tie order decides."""
    c = O.row_costs(O.content("ties", 64, 100))
    assert ((c == c.min(1, keepdims=True)).sum(1) >= 4).sum() >= 30
    img = O.content("paeth_ties", 270, 1440)
    assert (O.filter_rows(img)[0] == 4).sum() > 100


@pytest.mark.parametrize("h,w", SHAPES + [(1080, 1920)], ids=lambda v: str(v))
def test_layout_does_not_depend_on_content(h, w):
    lay = P.layout(h, w)
    for img in (O.content("random", h, w), np.full((h, w, 3), 255, np.uint8), np.zeros((h, w, 3), np.uint8)):
        assert P.parse(_cv2(img)) == lay
    assert sum(lay.block_lens) == h * (3 * w + 1) and max(lay.block_lens) <= 65535
    assert sum(lay.chunk_lens) == 2 + 5 * len(lay.block_lens) + h * (3 * w + 1) + 4


def test_plan_header_matches_the_layout():
    h, w = 270, 1440
    lay = P.layout(h, w)
    plan = N.PngPlan.from_buffer_copy(P.host_plan(h, w))
    assert (plan.H, plan.W, plan.n_blocks, plan.n_chunks) == (h, w, len(lay.block_lens), len(lay.chunk_lens))
    assert plan.file_bytes == len(_cv2(np.zeros((h, w, 3), np.uint8)))
    assert plan.max_chunk == max(lay.chunk_lens) and bytes(plan.zlib_header[:2]) == lay.zlib_header
    assert N.lib().b200_png_workspace_bytes(h, w) >= h * (3 * w + 1) + 8 * h


def _refused(lay, h, w, match, capacity=None):
    with pytest.raises(N.B200Error, match=match):
        if capacity is None:
            P.host_plan(h, w, lay)
        else:
            buf = (C.c_uint8 * capacity)()
            N.check(N.lib().b200_png_plan(h, w, lay.zlib_header, P._arr(lay.block_heads, C.c_uint8),
                                          P._arr(lay.block_lens, C.c_int32), len(lay.block_lens),
                                          P._arr(lay.chunk_lens, C.c_int32), len(lay.chunk_lens), lay.prefix,
                                          len(lay.prefix), lay.suffix, len(lay.suffix), buf, capacity), "b200_png_plan")


def test_plan_refuses_inconsistent_layouts():
    h, w = 5, 21846
    lay = P.layout(h, w)
    assert len(lay.block_lens) >= 2
    bl, cl = list(lay.block_lens), list(lay.chunk_lens)
    # a stored block over 65535 bytes (the next one shortened so the sum still matches)
    over = bl[:]
    over[0], over[1] = 65536, over[1] - (65536 - over[0])
    _refused(lay._replace(block_lens=tuple(over)), h, w, "at most 65535")
    # blocks that do not cover the filtered rows
    _refused(lay._replace(block_lens=tuple(bl[:-1] + [bl[-1] - 1])), h, w, "stored blocks hold")
    # chunks that do not cover the zlib stream
    _refused(lay._replace(chunk_lens=tuple(cl[:-1] + [cl[-1] + 1])), h, w, "IDAT chunks hold")
    # a BFINAL flag before the last block, a layout of another shape, not a zlib header, no IEND
    _refused(lay._replace(block_heads=(1,) + lay.block_heads[1:]), h, w, "BFINAL")
    _refused(lay, h, w + 1, "IHDR")
    _refused(lay._replace(zlib_header=b"\x78\x02"), h, w, "zlib header")
    _refused(lay._replace(suffix=lay.suffix[:-12]), h, w, "IEND")
    # a plan buffer that is too small
    need = N.lib().b200_png_plan_bytes(len(bl), len(cl), len(lay.prefix), len(lay.suffix))
    assert need > 0
    _refused(lay, h, w, "capacity", capacity=need - 8)
    assert len(P.host_plan(h, w, lay)) == need


def test_encode_refuses_before_touching_memory():
    """Argument errors of b200_png_encode are reported on the host, before any launch."""
    h, w = 17, 5
    data = P.host_plan(h, w)
    plan = N.PngPlan.from_buffer_copy(data)
    lib = N.lib()
    ws = lib.b200_png_workspace_bytes(h, w)
    fake = C.c_void_p(1 << 20)                         # never dereferenced: every call below fails validation
    assert lib.b200_png_encode(C.byref(plan), fake, fake, fake, ws, fake, plan.file_bytes - 1, None) != 0
    assert b"output capacity" in lib.b200_last_error()
    assert lib.b200_png_encode(C.byref(plan), fake, fake, fake, ws - 1, fake, plan.file_bytes, None) != 0
    assert b"workspace" in lib.b200_last_error()
    bad = N.PngPlan.from_buffer_copy(data)
    bad.magic = 0
    assert lib.b200_png_encode(C.byref(bad), fake, fake, fake, ws, fake, plan.file_bytes, None) != 0
    assert b"not a plan" in lib.b200_last_error()
    assert lib.b200_png_encode(C.byref(plan), None, fake, fake, ws, fake, plan.file_bytes, None) != 0
    assert b"null" in lib.b200_last_error()
    assert lib.b200_png_workspace_bytes(0, 5) == -1
