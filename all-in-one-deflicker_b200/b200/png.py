"""PNG encoding on the device: an 8-bit BGR image in, the bytes cv2.imwrite(path, img, [cv2.IMWRITE_PNG_COMPRESSION, 0])
writes out (save_img of src/models/utils.py), computed by b200_png_encode (csrc/png_encode.cu).

At compression level 0 the writer's file is libpng's adaptive row filters over zlib *stored* blocks.  What depends on
the pixels (filters, filtered bytes, Adler-32, IDAT CRCs) is computed on the device; what depends on the shape only
(zlib header, stored-block and IDAT lengths, the chunks around the IDATs) is read once per shape from the installed
OpenCV's own file of a blank image (`layout`), so the files stay equal to what that writer produces.
"""
from __future__ import annotations

import ctypes as C
import functools
import struct
from typing import NamedTuple

import numpy as np
import torch

from . import _native as N


class Layout(NamedTuple):
    """The shape-only parts of the writer's file of an (H, W, 3) image."""
    prefix: bytes           # signature, IHDR, any chunk before the first IDAT
    zlib_header: bytes      # CMF, FLG
    block_heads: tuple      # first byte of each stored block (BFINAL on the last)
    block_lens: tuple       # LEN of each stored block
    chunk_lens: tuple       # length of each IDAT chunk
    suffix: bytes           # the chunks after the last IDAT (IEND)


def parse(data: bytes) -> Layout:
    """Layout of a PNG file written with stored deflate blocks; raises ValueError on anything else."""
    if data[:8] != b"\x89PNG\r\n\x1a\n":
        raise ValueError("not a PNG file")
    p, prefix, chunk_lens, idat, after = 8, None, [], bytearray(), None
    while p < len(data):
        n, tag = struct.unpack(">I", data[p:p + 4])[0], data[p + 4:p + 8]
        if tag == b"IDAT":
            if after is not None:
                raise ValueError("IDAT chunks are not consecutive")
            if prefix is None:
                prefix = data[:p]
            chunk_lens.append(n)
            idat += data[p + 8:p + 8 + n]
        elif prefix is not None and after is None:
            after = p
        p += 12 + n
    if prefix is None or after is None:
        raise ValueError("no IDAT chunk, or nothing after it")
    q, heads, lens = 2, [], []
    while True:
        head = idat[q]
        if head & 6:
            raise ValueError("a deflate block that is not stored")
        ln, nln = struct.unpack("<HH", idat[q + 1:q + 5])
        if ln ^ nln != 0xFFFF:
            raise ValueError("stored block with NLEN != ~LEN")
        heads.append(head)
        lens.append(ln)
        q += 5 + ln
        if head & 1:
            break
    if q + 4 != len(idat):
        raise ValueError("bytes after the final stored block")
    return Layout(bytes(prefix), bytes(idat[:2]), tuple(heads), tuple(lens), tuple(chunk_lens), bytes(data[after:]))


@functools.lru_cache(maxsize=None)
def layout(h: int, w: int) -> Layout:
    """Layout of the installed OpenCV's level-0 PNG of an (h, w, 3) uint8 image, taken from a blank image's file."""
    import cv2
    ok, buf = cv2.imencode(".png", np.zeros((h, w, 3), np.uint8), [cv2.IMWRITE_PNG_COMPRESSION, 0])
    if not ok:
        raise N.B200Error("cv2.imencode failed on a blank %dx%d image" % (h, w))
    return parse(buf.tobytes())


def _arr(t, ctype):
    return (ctype * len(t))(*t)


def host_plan(h: int, w: int, lay: Layout | None = None) -> bytes:
    """The plan b200_png_encode reads, built and validated by b200_png_plan (host only)."""
    lay = layout(h, w) if lay is None else lay
    lib = N.lib()
    size = lib.b200_png_plan_bytes(len(lay.block_lens), len(lay.chunk_lens), len(lay.prefix), len(lay.suffix))
    if size < 0:
        raise N.B200Error("b200_png_plan_bytes: " + N.last_error())
    buf = (C.c_uint8 * size)()
    N.check(lib.b200_png_plan(h, w, lay.zlib_header, _arr(lay.block_heads, C.c_uint8), _arr(lay.block_lens, C.c_int32),
                              len(lay.block_lens), _arr(lay.chunk_lens, C.c_int32), len(lay.chunk_lens), lay.prefix,
                              len(lay.prefix), lay.suffix, len(lay.suffix), buf, size), "b200_png_plan")
    return bytes(buf)


class Plan:
    """One shape's plan: the host header b200_png_encode checks and the uploaded copy its kernels read."""

    def __init__(self, h: int, w: int, device):
        data = host_plan(h, w)
        self.header = N.PngPlan.from_buffer_copy(data)
        self.device = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(device)
        self.file_bytes = int(self.header.file_bytes)
        self.workspace_bytes = int(N.lib().b200_png_workspace_bytes(h, w))


@functools.lru_cache(maxsize=None)
def _plan(h: int, w: int, device: torch.device) -> Plan:
    return Plan(h, w, device)


def plan(h: int, w: int, device) -> Plan:
    """The cached plan of an (h, w, 3) image on `device` (built and uploaded on first use)."""
    device = torch.device(device)
    if device.index is None:
        device = torch.device(device.type, torch.cuda.current_device())
    return _plan(h, w, device)


def encode(img, out=None, workspace=None):
    """PNG file of the contiguous uint8 BGR CUDA image `img` (H, W, 3), as a uint8 CUDA tensor of the file's length
    (a view of `out` when given).  Stream-ordered on the current stream; nothing is allocated when `out` and
    `workspace` are given and the shape's plan exists, so it can be captured in a CUDA graph after one call."""
    if not (torch.is_tensor(img) and img.is_cuda and img.dtype == torch.uint8 and img.is_contiguous() and img.dim() == 3
            and img.shape[2] == 3):
        raise N.B200Error("png.encode takes a contiguous uint8 CUDA image (H, W, 3)")
    h, w = img.shape[:2]
    p = plan(h, w, img.device)
    if workspace is None:
        workspace = torch.empty(p.workspace_bytes, dtype=torch.uint8, device=img.device)
    if out is None:
        out = torch.empty(p.file_bytes, dtype=torch.uint8, device=img.device)
    for t, what in ((workspace, "workspace"), (out, "out")):
        if not (t.is_cuda and t.dtype == torch.uint8 and t.is_contiguous() and t.device == img.device):
            raise N.B200Error("png.encode: %s must be a contiguous uint8 tensor on the image's device" % what)
    N.check(N.lib().b200_png_encode(C.byref(p.header), N.ptr(p.device), N.ptr(img), N.ptr(workspace), workspace.numel(),
                                    N.ptr(out), out.numel(), N.current_stream()), "b200_png_encode")
    return out[:p.file_bytes]
