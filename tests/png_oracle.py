"""CPU restatement of OpenCV's level-0 PNG writer for 8-bit BGR images (cv2.imwrite(path, img,
[cv2.IMWRITE_PNG_COMPRESSION, 0]): libpng's adaptive row filters, zlib stored blocks), the reference b200_png_encode
is tested against.

libpng's choice, per row of the RGB bytes (OpenCV hands BGR to libpng with png_set_bgr): for None, Sub, Up, Average and
Paeth in that order, the cost is the sum over the filtered bytes v of min(v, 256 - v); the first smallest cost wins;
row 0's previous row is zeros.  libpng drops, before it starts, the filters that would read a neighbour the image does
not have: Up, Average and Paeth when the image has one row, Sub, Average and Paeth when it has one column.  The file is
then the shape's layout (b200.png.Layout) around the filtered stream, with zlib's Adler-32 and the IDATs' CRC-32 from
the zlib module."""
import struct
import zlib

import numpy as np

FILTERS = ("none", "sub", "up", "average", "paeth")


def _candidates(rows, prev):
    """The five filtered versions (5, n, R) of the RGB rows (n, R) given their previous rows, as int32 in [0, 256)."""
    z = np.zeros((rows.shape[0], 3), np.int32)
    a = np.concatenate([z, rows[:, :-3]], axis=1)
    b = prev
    c = np.concatenate([z, prev[:, :-3]], axis=1)
    pa, pb, pc = np.abs(b - c), np.abs(a - c), np.abs(a + b - 2 * c)             # libpng's png_setup_paeth_row
    paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    return np.stack([rows, rows - a, rows - b, rows - ((a + b) >> 1), rows - paeth]) & 255


def allowed(h, w):
    """The filters libpng tries for an (h, w) image, as a boolean mask over FILTERS."""
    m = np.ones(5, bool)
    if h == 1:
        m[[2, 3, 4]] = False
    if w == 1:
        m[[1, 3, 4]] = False
    return m


def row_costs(img, batch=64):
    """(H, 5) int64: each row's cost under each filter (filters libpng does not try for the shape cost 2^62)."""
    rgb = np.ascontiguousarray(img[..., ::-1]).reshape(img.shape[0], -1).astype(np.int32)
    prev = np.concatenate([np.zeros_like(rgb[:1]), rgb[:-1]])
    out = []
    for y in range(0, rgb.shape[0], batch):
        v = _candidates(rgb[y:y + batch], prev[y:y + batch])
        out.append(np.minimum(v, 256 - v).sum(axis=2, dtype=np.int64).T)
    return np.where(allowed(*img.shape[:2]), np.concatenate(out), np.int64(1) << 62)


def filter_rows(img, batch=64):
    """(filters (H,) uint8, raw stream bytes: each row's filter byte then its filtered bytes) of a uint8 BGR image."""
    h = img.shape[0]
    rgb = np.ascontiguousarray(img[..., ::-1]).reshape(h, -1).astype(np.int32)
    prev = np.concatenate([np.zeros_like(rgb[:1]), rgb[:-1]])
    filters = np.empty(h, np.uint8)
    raw = np.empty((h, rgb.shape[1] + 1), np.uint8)
    for y in range(0, h, batch):
        v = _candidates(rgb[y:y + batch], prev[y:y + batch])
        cost = np.minimum(v, 256 - v).sum(axis=2, dtype=np.int64)
        cost[~allowed(*img.shape[:2])] = np.int64(1) << 62
        f = np.argmin(cost, axis=0)                                               # the first minimum: ties go low
        filters[y:y + batch] = f
        raw[y:y + batch, 0] = f
        raw[y:y + batch, 1:] = v[f, np.arange(len(f))]
    return filters, raw.tobytes()


def assemble(raw, lay):
    """The file: lay.prefix, the zlib stream of stored blocks cut into IDAT chunks, lay.suffix."""
    z, q = bytearray(lay.zlib_header), 0
    for head, n in zip(lay.block_heads, lay.block_lens):
        z += bytes([head]) + struct.pack("<HH", n, n ^ 0xFFFF) + raw[q:q + n]
        q += n
    assert q == len(raw), "the layout's blocks do not cover the stream"
    z += struct.pack(">I", zlib.adler32(raw))
    out, q = bytearray(lay.prefix), 0
    for n in lay.chunk_lens:
        data = bytes(z[q:q + n])
        out += struct.pack(">I", n) + b"IDAT" + data + struct.pack(">I", zlib.crc32(b"IDAT" + data))
        q += n
    assert q == len(z), "the layout's chunks do not cover the stream"
    return bytes(out + lay.suffix)


def encode(img, lay):
    return assemble(filter_rows(img)[1], lay)


def idat_filters(data, h, w):
    """Filter byte of each row of a level-0 PNG file of an (h, w, 3) image (inflated with zlib)."""
    p, idat = 8, b""
    while p < len(data):
        n = struct.unpack(">I", data[p:p + 4])[0]
        if data[p + 4:p + 8] == b"IDAT":
            idat += data[p + 8:p + 8 + n]
        p += 12 + n
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 3 * w + 1)
    return raw[:, 0].copy()


# ---- test images -----------------------------------------------------------------------------------------------------
def content(kind, h, w, seed=0):
    """uint8 BGR (h, w, 3) test images by name."""
    rng = np.random.default_rng(seed + 7919 * h + w)
    if kind == "random":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "gradient":
        yy, xx = np.mgrid[0:h, 0:w]
        return np.stack([(xx * 3 + yy) % 256, (xx + 2 * yy) % 256, (xx * 255 // max(w - 1, 1)) % 256], -1).astype(np.uint8)
    if kind.startswith("const"):
        return np.full((h, w, 3), int(kind[5:]), np.uint8)
    if kind == "ties":
        # odd rows are a smooth random walk x, even rows are x shifted right by one pixel behind a black pixel, so on odd
        # rows Sub, Up, Average and Paeth all leave the same bytes: the smallest cost is shared by four filters
        x = np.cumsum(rng.integers(-2, 3, (h, w, 3)), axis=1) + rng.integers(0, 256, (h, 1, 3))
        for y in range(0, h - 1, 2):
            x[y, 0], x[y, 1:] = 0, x[y + 1, :-1]
        return (x & 255).astype(np.uint8)
    if kind == "paeth_ties":
        # up and up-left equal, left a step away, and steps of 2: |b - c|, |a - c|, |a + b - 2c| meet often, and the
        # rows move so that Paeth is picked on some of them
        base = rng.integers(0, 3, (h, w, 3)) * 2
        return np.cumsum(np.cumsum(base, axis=0), axis=1).astype(np.uint8)
    raise ValueError(kind)


KINDS = ("random", "gradient", "const0", "const128", "const255", "ties", "paeth_ties")
