// PNG encoding of stage 2's output frames on the device (DESIGN §4b): an 8-bit BGR image (H, W, 3) in, the file
// cv2.imwrite(path, img, [IMWRITE_PNG_COMPRESSION, 0]) writes out, byte for byte.
//
// At compression level 0 OpenCV's writer (libpng + zlib) produces: signature and IHDR, a zlib stream of *stored*
// deflate blocks cut into IDAT chunks, IEND.  Only three things depend on the pixels: each row's filter (libpng's
// adaptive choice), the filtered bytes, and the checksums (the stream's Adler-32, one CRC-32 per chunk).  Everything
// else — the zlib header, the stored-block lengths, the chunk lengths, the bytes around the IDAT chunks — depends on
// (H, W) only and comes from the caller as a plan (b200_png_plan; b200/png.py takes it from OpenCV's file of a blank
// image of the same shape).
//
//   png_filter_kernel    one CTA per row: libpng's filter choice on the RGB row (OpenCV hands BGR to libpng with
//                        png_set_bgr; the cost of a filter is the sum of min(v, 256 - v) over the filtered bytes v, the
//                        first smallest wins, row 0's previous row is zeros), the filtered row with its filter byte into the raw stream, and the row's
//                        Adler-32 partial sums
//   png_assemble_kernel  one CTA per IDAT chunk: length, tag, the chunk's slice of the zlib stream (header, stored-block
//                        headers, raw bytes, Adler-32 trailer), CRC-32 of tag + data; one more CTA writes the bytes
//                        before the first chunk and after the last
#include "common.cuh"

#include <cstring>

namespace b200 {

constexpr int kPngThreads = 256;
constexpr int kCrcLanes = 64;              // threads of an assembly CTA that compute the chunk's CRC
constexpr uint32_t kAdlerMod = 65521;
constexpr uint32_t kCrcPoly = 0xedb88320u;  // CRC-32 (ISO 3309), reflected

// libpng's filter types, in the order its adaptive choice tries them (ties go to the earlier one)
enum { F_NONE = 0, F_SUB = 1, F_UP = 2, F_AVG = 3, F_PAETH = 4 };

__device__ __forceinline__ uint32_t filter_cost(uint32_t v) { return v < 128 ? v : 256 - v; }

// predictor of filter f for one byte: a = left (same channel, previous pixel), b = up, c = up-left; 0 outside the image
__device__ __forceinline__ uint32_t png_predict(int f, int a, int b, int c) {
  switch (f) {
    case F_SUB: return a;
    case F_UP: return b;
    case F_AVG: return (a + b) >> 1;
    case F_PAETH: {
      const int pa = abs(b - c), pb = abs(a - c), pc = abs(a + b - 2 * c);     // libpng's png_setup_paeth_row
      return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
    }
    default: return 0;
  }
}

// byte i of the RGB row (x, a, b, c) read from the BGR image rows cur / prev (prev == nullptr on row 0)
struct Taps { int x, a, b, c; };
__device__ __forceinline__ Taps png_taps(const uint8_t* __restrict__ cur, const uint8_t* __restrict__ prev, int i) {
  const int p = i / 3, src = 3 * p + 2 - (i - 3 * p);
  Taps t;
  t.x = __ldg(cur + src);
  t.a = i >= 3 ? __ldg(cur + src - 3) : 0;
  t.b = prev ? __ldg(prev + src) : 0;
  t.c = (prev && i >= 3) ? __ldg(prev + src - 3) : 0;
  return t;
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

__global__ void __launch_bounds__(kPngThreads) png_filter_kernel(const uint8_t* __restrict__ img, int H, int W,
                                                                 uint8_t* __restrict__ raw,
                                                                 uint32_t* __restrict__ adler_rows) {
  constexpr int kWarps = kPngThreads / 32;
  __shared__ uint32_t s_cost[kWarps][5];
  __shared__ uint64_t s_adler[kWarps][2];
  __shared__ int s_filter;
  const int y = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int R = 3 * W;
  const int64_t L = R + 1;
  const uint8_t* cur = img + (int64_t)y * R;
  const uint8_t* prev = y > 0 ? cur - R : nullptr;

  uint32_t cost[5] = {0, 0, 0, 0, 0};
  for (int i = threadIdx.x; i < R; i += kPngThreads) {
    const Taps t = png_taps(cur, prev, i);
#pragma unroll
    for (int f = 0; f < 5; ++f) cost[f] += filter_cost((uint32_t)(t.x - (int)png_predict(f, t.a, t.b, t.c)) & 0xff);
  }
#pragma unroll
  for (int f = 0; f < 5; ++f) {
    const uint32_t s = warp_sum(cost[f]);
    if (lane == 0) s_cost[warp][f] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // libpng leaves out the filters that read a neighbour the image does not have (png_write_start_row)
    unsigned tried = 0x1f;
    if (H == 1) tried &= ~(1u << F_UP | 1u << F_AVG | 1u << F_PAETH);
    if (W == 1) tried &= ~(1u << F_SUB | 1u << F_AVG | 1u << F_PAETH);
    int best = 0;
    uint32_t best_cost = 0;
    for (int f = 0; f < 5; ++f) {
      uint32_t s = 0;
      for (int w = 0; w < kWarps; ++w) s += s_cost[w][f];
      if (f == 0 || ((tried >> f & 1) && s < best_cost)) best = f, best_cost = s;   // strictly smaller: ties go low
    }
    s_filter = best;
  }
  __syncthreads();
  const int f = s_filter;

  // the filtered row, and its Adler-32 partials: s1 = sum of bytes, s2 = sum of bytes weighted by their distance to
  // the row's end (the last byte weighs 1), combined over rows by the assembly kernel
  uint8_t* out = raw + (int64_t)y * L;
  uint64_t s1 = 0, s2 = 0;
  for (int i = threadIdx.x; i < R; i += kPngThreads) {
    const Taps t = png_taps(cur, prev, i);
    const uint32_t v = (uint32_t)(t.x - (int)png_predict(f, t.a, t.b, t.c)) & 0xff;
    out[1 + i] = (uint8_t)v;
    s1 += v;
    s2 += (uint64_t)(L - 1 - i) * v;
  }
  if (threadIdx.x == 0) {
    out[0] = (uint8_t)f;
    s1 += f;
    s2 += (uint64_t)L * f;
  }
  s1 = warp_sum(s1);
  s2 = warp_sum(s2);
  if (lane == 0) s_adler[warp][0] = s1, s_adler[warp][1] = s2;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t a = 0, b = 0;
    for (int w = 0; w < kWarps; ++w) a += s_adler[w][0], b += s_adler[w][1];
    adler_rows[2 * y] = (uint32_t)(a % kAdlerMod);
    adler_rows[2 * y + 1] = (uint32_t)(b % kAdlerMod);
  }
}

// a(x) * b(x) mod P(x), reflected (zlib's multmodp)
__device__ __forceinline__ uint32_t crc_multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return p;
}

// x^(8 n) mod P(x) from x2n[k] = x^(2^k) mod P(x)
__device__ __forceinline__ uint32_t crc_shift(const uint32_t* x2n, uint32_t n) {
  uint32_t p = 1u << 31;                    // x^0
  for (int k = 3; n; n >>= 1, ++k)
    if (n & 1) p = crc_multmodp(x2n[k & 31], p);
  return p;
}

__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
  p[0] = (uint8_t)(v >> 24), p[1] = (uint8_t)(v >> 16), p[2] = (uint8_t)(v >> 8), p[3] = (uint8_t)v;
}

struct PngTables {
  const uint32_t* block_raw;    // [n_blocks + 1] raw-stream offset of each stored block; the last entry = raw_bytes
  const uint32_t* chunk_z;      // [n_chunks + 1] zlib-stream offset of each IDAT chunk; the last entry = zlib_bytes
  const uint8_t* prefix;
  const uint8_t* suffix;
};

__device__ __forceinline__ uint32_t block_z(const uint32_t* block_raw, int b) { return 2 + 5u * b + block_raw[b]; }

__global__ void __launch_bounds__(kPngThreads) png_assemble_kernel(B200PngPlan p, PngTables tab,
                                                                   const uint8_t* __restrict__ raw,
                                                                   const uint32_t* __restrict__ adler_rows,
                                                                   uint8_t* __restrict__ out) {
  extern __shared__ __align__(16) uint8_t s_chunk[];     // "IDAT" + data, max_chunk + 4 bytes (+ 4 of padding)
  __shared__ uint32_t s_crc_table[256];
  __shared__ uint32_t s_x2n[32];
  __shared__ uint64_t s_red[kPngThreads / 32][2];
  __shared__ uint32_t s_adler;
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (c == p.n_chunks) {                                  // signature, IHDR / IEND
    for (int i = tid; i < p.prefix_bytes; i += kPngThreads) out[i] = tab.prefix[i];
    uint8_t* tail = out + p.file_bytes - p.suffix_bytes;
    for (int i = tid; i < p.suffix_bytes; i += kPngThreads) tail[i] = tab.suffix[i];
    return;
  }

  const uint32_t z0 = tab.chunk_z[c], n = tab.chunk_z[c + 1] - z0;
  const uint32_t trailer = (uint32_t)p.zlib_bytes - 4;
  uint8_t* o = out + p.prefix_bytes + 12ll * c + z0;

  if (z0 + n > trailer) {                                 // this chunk holds (part of) the Adler-32 trailer
    const uint64_t L = 3ull * p.W + 1;
    uint64_t a = 0, b = 0;
    for (int y = tid; y < p.H; y += kPngThreads) {
      const uint64_t s1 = adler_rows[2 * y], s2 = adler_rows[2 * y + 1];
      a += s1;
      b += s2 + s1 * (((uint64_t)(p.H - 1 - y) * L) % kAdlerMod);
    }
    a = warp_sum(a);
    b = warp_sum(b);
    if (lane == 0) s_red[warp][0] = a, s_red[warp][1] = b;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < kPngThreads / 32; ++w) a += s_red[w][0], b += s_red[w][1];
      a = (1 + a) % kAdlerMod;
      b = ((uint64_t)p.raw_bytes % kAdlerMod + b) % kAdlerMod;
      s_adler = (uint32_t)(b << 16 | a);
    }
    __syncthreads();
  }

  for (int i = tid; i < 256; i += kPngThreads) {
    uint32_t v = i;
    for (int k = 0; k < 8; ++k) v = (v & 1) ? (v >> 1) ^ kCrcPoly : v >> 1;
    s_crc_table[i] = v;
  }
  if (tid == 0) {
    uint32_t v = 1u << 30;                                // x^1
    for (int k = 0; k < 32; ++k) s_x2n[k] = v, v = crc_multmodp(v, v);
  }

  // the chunk's bytes of the zlib stream; each thread walks its bytes in increasing order with a block cursor
  int blk = 0;
  {
    const uint32_t z = z0 + tid;
    if (z >= 2 && z < trailer) {                          // last block starting at or before z
      int lo = 0, hi = p.n_blocks;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (block_z(tab.block_raw, mid) <= z) lo = mid; else hi = mid;
      }
      blk = lo;
    }
  }
  for (uint32_t j = tid; j < n; j += kPngThreads) {
    const uint32_t z = z0 + j;
    uint8_t v;
    if (z < 2) {
      v = z == 0 ? p.zlib_header[0] : p.zlib_header[1];
    } else if (z >= trailer) {
      v = (uint8_t)(s_adler >> (8 * (3 - (z - trailer))));
    } else {
      while (block_z(tab.block_raw, blk + 1) <= z) ++blk;
      const uint32_t r0 = tab.block_raw[blk], off = z - (2 + 5u * blk + r0);
      const uint32_t len = tab.block_raw[blk + 1] - r0;
      switch (off) {
        case 0: v = blk == p.n_blocks - 1; break;         // BFINAL, BTYPE 00 (stored)
        case 1: v = (uint8_t)len; break;                  // LEN, little-endian
        case 2: v = (uint8_t)(len >> 8); break;
        case 3: v = (uint8_t)~len; break;                 // NLEN = ~LEN
        case 4: v = (uint8_t)(~len >> 8); break;
        default: v = raw[r0 + off - 5];
      }
    }
    s_chunk[4 + j] = v;
    o[8 + j] = v;
  }
  if (tid < 4) {
    const uint8_t tag = (uint8_t)(0x49444154u >> (8 * (3 - tid)));      // "IDAT"
    s_chunk[tid] = tag;
    o[4 + tid] = tag;
    o[tid] = (uint8_t)(n >> (8 * (3 - tid)));
  }
  __syncthreads();

  // CRC-32 of tag + data: lane t takes a run of `seg` bytes (a multiple of 4 with seg / 4 odd, so the word reads of a
  // warp fall in distinct banks), computes its CRC from a zero register, and shifts it past the bytes after its run;
  // the XOR of the lanes' terms is the CRC from zero of the whole, and the standard initial value ~0 adds x^(8N) * ~0
  if (warp < kCrcLanes / 32) {
    const uint32_t N = n + 4;
    uint32_t seg = ((N + kCrcLanes - 1) / kCrcLanes + 3) & ~3u;
    if (!((seg >> 2) & 1)) seg += 4;
    const uint32_t begin = min(tid * seg, N), end = min(begin + seg, N);
    uint32_t crc = 0, i = begin;
    for (; i + 4 <= end; i += 4) {
      const uint32_t w = *reinterpret_cast<const uint32_t*>(s_chunk + i);
#pragma unroll
      for (int k = 0; k < 4; ++k) crc = s_crc_table[(crc ^ (w >> (8 * k))) & 0xff] ^ (crc >> 8);
    }
    for (; i < end; ++i) crc = s_crc_table[(crc ^ s_chunk[i]) & 0xff] ^ (crc >> 8);
    uint32_t term = end > begin ? crc_multmodp(crc_shift(s_x2n, N - end), crc) : 0;
    for (int d = 16; d > 0; d >>= 1) term ^= __shfl_xor_sync(0xffffffffu, term, d);
    if (lane == 0) s_red[warp][0] = term;
  }
  __syncthreads();
  if (tid == 0) {
    const uint32_t N = n + 4;
    uint32_t all = crc_multmodp(crc_shift(s_x2n, N), 0xffffffffu);
    for (int w = 0; w < kCrcLanes / 32; ++w) all ^= (uint32_t)s_red[w][0];
    put_be32(o + 8 + n, ~all);
  }
}

// plan tables, 8-byte aligned, after the header
inline int64_t align8(int64_t v) { return (v + 7) & ~int64_t(7); }

}  // namespace b200

using namespace b200;

extern "C" {

int64_t b200_png_plan_bytes(int32_t n_blocks, int32_t n_chunks, int32_t prefix_bytes, int32_t suffix_bytes) {
  if (n_blocks < 1 || n_chunks < 1 || prefix_bytes < 0 || suffix_bytes < 0 || prefix_bytes > B200_PNG_MAX_PREFIX ||
      suffix_bytes > B200_PNG_MAX_PREFIX || n_blocks > (1 << 24) || n_chunks > (1 << 24)) {
    set_error("png plan: bad table sizes (%d blocks, %d chunks, %d + %d bytes around them)", n_blocks, n_chunks,
              prefix_bytes, suffix_bytes);
    return -1;
  }
  return align8(sizeof(B200PngPlan)) + align8(4ll * (n_blocks + 1)) + align8(4ll * (n_chunks + 1)) +
         align8(prefix_bytes) + align8(suffix_bytes);
}

int b200_png_plan(int32_t H, int32_t W, const uint8_t* zlib_header, const uint8_t* block_heads,
                  const int32_t* block_lens, int32_t n_blocks, const int32_t* chunk_lens, int32_t n_chunks,
                  const uint8_t* prefix, int32_t prefix_bytes, const uint8_t* suffix, int32_t suffix_bytes, void* plan,
                  int64_t plan_capacity) {
  B200_REQUIRE(zlib_header && block_heads && block_lens && chunk_lens && prefix && suffix && plan, "null pointer");
  B200_REQUIRE(H > 0 && W > 0, "png plan: bad image size %dx%d", H, W);
  const int64_t raw_bytes = (int64_t)H * (3ll * W + 1);
  B200_REQUIRE(raw_bytes <= B200_PNG_MAX_RAW, "png plan: %dx%d has %lld filtered bytes, more than %lld", H, W,
               (long long)raw_bytes, (long long)B200_PNG_MAX_RAW);
  const int64_t need = b200_png_plan_bytes(n_blocks, n_chunks, prefix_bytes, suffix_bytes);
  if (need < 0) return B200_ERR_INVALID;
  B200_REQUIRE(plan_capacity >= need, "png plan: capacity %lld bytes, the plan needs %lld", (long long)plan_capacity,
               (long long)need);

  static const uint8_t kSignature[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  B200_REQUIRE(prefix_bytes >= 33 && memcmp(prefix, kSignature, 8) == 0 && memcmp(prefix + 12, "IHDR", 4) == 0,
               "png plan: the prefix does not start with the PNG signature and IHDR");
  auto be32 = [](const uint8_t* q) { return (uint32_t)q[0] << 24 | (uint32_t)q[1] << 16 | (uint32_t)q[2] << 8 | q[3]; };
  B200_REQUIRE(be32(prefix + 16) == (uint32_t)W && be32(prefix + 20) == (uint32_t)H && prefix[24] == 8 &&
                   prefix[25] == 2 && prefix[28] == 0,
               "png plan: IHDR is not a non-interlaced 8-bit RGB image of %dx%d", H, W);
  B200_REQUIRE(suffix_bytes >= 12 && memcmp(suffix + suffix_bytes - 8, "IEND", 4) == 0,
               "png plan: the suffix does not end with IEND");
  B200_REQUIRE((zlib_header[0] & 0x0f) == 8 && (zlib_header[0] >> 4) <= 7 && !(zlib_header[1] & 0x20) &&
                   ((zlib_header[0] << 8) | zlib_header[1]) % 31 == 0,
               "png plan: %02x%02x is not a zlib header", zlib_header[0], zlib_header[1]);

  int64_t sum = 0;
  for (int32_t b = 0; b < n_blocks; ++b) {
    B200_REQUIRE(block_lens[b] >= 0 && block_lens[b] <= 65535, "png plan: stored block %d has %d bytes (at most 65535)",
                 b, block_lens[b]);
    B200_REQUIRE(block_heads[b] == (b == n_blocks - 1 ? 1 : 0),
                 "png plan: block %d header byte %d (stored blocks; BFINAL on the last only)", b, block_heads[b]);
    sum += block_lens[b];
  }
  B200_REQUIRE(sum == raw_bytes, "png plan: stored blocks hold %lld bytes, %dx%d filters to %lld", (long long)sum, H, W,
               (long long)raw_bytes);
  const int64_t zlib_bytes = 2 + 5ll * n_blocks + raw_bytes + 4;
  int64_t zsum = 0;
  int32_t max_chunk = 0;
  for (int32_t c = 0; c < n_chunks; ++c) {
    B200_REQUIRE(chunk_lens[c] > 0 && chunk_lens[c] <= B200_PNG_MAX_CHUNK,
                 "png plan: IDAT chunk %d has %d bytes (1 to %d)", c, chunk_lens[c], B200_PNG_MAX_CHUNK);
    zsum += chunk_lens[c];
    max_chunk = chunk_lens[c] > max_chunk ? chunk_lens[c] : max_chunk;
  }
  B200_REQUIRE(zsum == zlib_bytes, "png plan: IDAT chunks hold %lld bytes, the zlib stream has %lld", (long long)zsum,
               (long long)zlib_bytes);

  B200PngPlan h;
  memset(&h, 0, sizeof h);
  h.magic = B200_PNG_PLAN_MAGIC;
  h.H = H, h.W = W, h.n_blocks = n_blocks, h.n_chunks = n_chunks;
  h.prefix_bytes = prefix_bytes, h.suffix_bytes = suffix_bytes, h.max_chunk = max_chunk;
  h.raw_bytes = raw_bytes, h.zlib_bytes = zlib_bytes;
  h.file_bytes = prefix_bytes + 12ll * n_chunks + zlib_bytes + suffix_bytes;
  h.plan_bytes = need;
  h.zlib_header[0] = zlib_header[0], h.zlib_header[1] = zlib_header[1];
  h.block_raw_at = align8(sizeof(B200PngPlan));
  h.chunk_z_at = h.block_raw_at + align8(4ll * (n_blocks + 1));
  h.prefix_at = h.chunk_z_at + align8(4ll * (n_chunks + 1));
  h.suffix_at = h.prefix_at + align8(prefix_bytes);

  uint8_t* base = static_cast<uint8_t*>(plan);
  memset(base, 0, need);
  memcpy(base, &h, sizeof h);
  uint32_t* block_raw = reinterpret_cast<uint32_t*>(base + h.block_raw_at);
  uint32_t* chunk_z = reinterpret_cast<uint32_t*>(base + h.chunk_z_at);
  block_raw[0] = 0;
  for (int32_t b = 0; b < n_blocks; ++b) block_raw[b + 1] = block_raw[b] + (uint32_t)block_lens[b];
  chunk_z[0] = 0;
  for (int32_t c = 0; c < n_chunks; ++c) chunk_z[c + 1] = chunk_z[c] + (uint32_t)chunk_lens[c];
  memcpy(base + h.prefix_at, prefix, prefix_bytes);
  memcpy(base + h.suffix_at, suffix, suffix_bytes);
  return B200_OK;
}

int64_t b200_png_workspace_bytes(int32_t H, int32_t W) {
  if (H <= 0 || W <= 0 || (int64_t)H * (3ll * W + 1) > B200_PNG_MAX_RAW) {
    set_error("png workspace: bad image size %dx%d", H, W);
    return -1;
  }
  return align8((int64_t)H * (3ll * W + 1)) + 8ll * H;
}

int b200_png_encode(const B200PngPlan* plan, const void* plan_device, const uint8_t* image, void* workspace,
                    int64_t workspace_bytes, uint8_t* out, int64_t out_capacity, void* stream) {
  B200_REQUIRE(plan && plan_device && image && workspace && out, "null pointer");
  B200_REQUIRE(plan->magic == B200_PNG_PLAN_MAGIC, "png encode: not a plan made by b200_png_plan");
  const int64_t ws = b200_png_workspace_bytes(plan->H, plan->W);
  if (ws < 0) return B200_ERR_INVALID;
  B200_REQUIRE(workspace_bytes >= ws, "png encode: workspace of %lld bytes, %dx%d needs %lld",
               (long long)workspace_bytes, plan->H, plan->W, (long long)ws);
  B200_REQUIRE(out_capacity >= plan->file_bytes, "png encode: output capacity %lld bytes, the file has %lld",
               (long long)out_capacity, (long long)plan->file_bytes);
  B200_REQUIRE((reinterpret_cast<uintptr_t>(plan_device) & 7) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 7) == 0,
               "png encode: plan and workspace must be 8-byte aligned");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* raw = static_cast<uint8_t*>(workspace);
  uint32_t* adler_rows = reinterpret_cast<uint32_t*>(raw + align8(plan->raw_bytes));
  png_filter_kernel<<<plan->H, kPngThreads, 0, st>>>(image, plan->H, plan->W, raw, adler_rows);
  B200_CHECK_LAUNCH();
  const uint8_t* pd = static_cast<const uint8_t*>(plan_device);
  const PngTables tab{reinterpret_cast<const uint32_t*>(pd + plan->block_raw_at),
                      reinterpret_cast<const uint32_t*>(pd + plan->chunk_z_at), pd + plan->prefix_at,
                      pd + plan->suffix_at};
  png_assemble_kernel<<<plan->n_chunks + 1, kPngThreads, plan->max_chunk + 8, st>>>(*plan, tab, raw, adler_rows, out);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
