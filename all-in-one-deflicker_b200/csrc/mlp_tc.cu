// wgmma path of the two IMLPs (B200_PREC_TC).
//
// Every 256-wide Linear layer runs on the tensor cores (wgmma m64n256k16, fp16 operands, fp32 accumulators in the
// registers of a consumer warpgroup, 128-row CTA tiles split over two warpgroups).  fp32 fidelity comes from a 2-term
// fp16 split of BOTH operands,
//     v * S = hi + lo,   hi = rn_f16(v*S),  lo = rn_f16(v*S - hi)          (22-bit significand)
// and three MMAs per product  hi*hi + hi*lo + lo*hi  (the dropped lo*lo term is 2^-22 relative).
// S is a power of two per operand class (activations 2^4, weights 2^8, gradients chosen per
// iteration from max|dL/dy|), undone exactly in the epilogues.
//
// Kernels
//   tc_prep_kernel   fp32 parameters -> split fp16 weight items (16 KB each, the exact 64B-swizzled smem
//                    layout a wgmma descriptor reads), W for the forward and W^T for the dgrad
//   tc_fwd_kernel    persistent; one 128-row tile walks through ALL layers on chip: the A operand lives in
//                    shared memory in the image layout, weights stream L2->smem through the TMA engine
//                    (cp.async.bulk + mbarrier ring, one producer warp), the epilogue of each warpgroup
//                    (bias + ReLU + split) rewrites its rows of the A tile in place and bulk-stores them as the
//                    activation image the weight-gradient kernel consumes; first/last (K=3 / N=2,3) layers and the
//                    positional encoding run on CUDA cores inside the same kernel
//   tc_bwd_kernel    same structure for dL/dz: tanh', last layer on CUDA cores, hidden layers as
//                    dZ * W (B = W^T images), ReLU mask from 1-bit flags; bias gradients (and the mapping's dW0)
//                    as row sums of each dZ tile by m64n8k16 MMAs against a [1, x, y, t] operand
//   tc_wgrad_kernel  dW = dZ^T * H as wgmma with both operands MN-major straight from the images
//                    the two kernels above left in HBM; split over rows, fp32 vector reductions; clusters of two CTAs
//                    split the 256-wide operand and multicast the other, so each image byte is read once
//
// Networks (TcNet, one row of g_kernels each): the plain mappings (6 / 4 layers), the atlas, the alpha network and the
// position-encoded mappings (3 -> PE 1..10 -> 256 x {4,2} -> 2, use_positional_encoding_mapping1/2).
//
// Restates nn.Linear/ReLU/tanh/skip-concat forward+autograd of
//   src/models/stage_1/implicit_neural_networks.py:62-81 for the two networks of
//   src/stage1_neural_atlas.py:112-128.
#include <mutex>
#include <vector>

#include "tc_api.cuh"
#include "tc_ptx.cuh"
#include "loss_math.h"

namespace b200 {
using namespace ptx;

constexpr int TM = 128;                 // rows per tile
constexpr int HID = 256;
constexpr int ITEM_BYTES = 16384;       // one weight item: 256 rows x 32 k (fp16), K-major, 64B swizzle
constexpr int CHUNK_BYTES = 4 * ITEM_BYTES;   // one 64-wide k chunk of a weight: hi k 0-31, hi k 32-63, lo k 0-31, lo 32-63
constexpr float S_ACT = 16.0f;          // activation scale before the fp16 split
constexpr float S_W = 256.0f;           // weight scale
constexpr int ATOM_BYTES = TM * 128;    // one 64-column block of a tile image, one term: 16 KB
constexpr int TILE_IMG_BYTES = 4 * ATOM_BYTES;   // one term of one [128 x 256] activation tile image: 64 KB
constexpr int PE_COLS = 40;

// Tile image = 4 atom blocks (64 columns each); an atom block is [16 groups of 8 rows][8 rows x 128 B]
// with the 16-byte chunks of a row XOR-swizzled by (row & 7).  The same bytes are a K-major SW128 wgmma
// operand (M/N = rows, K = the 64 columns) and an MN-major SW128 operand (MN = columns, K = rows).
__host__ __device__ __forceinline__ int atom_off(int m, int k) {          // k in [0, 64)
  const int r = m & 7;
  return (m >> 3) * 1024 + r * 128 + (((k >> 3) ^ r) << 4) + ((k & 7) << 1);
}
// Weight item = [32 groups of 8 rows][8 rows x 64 B] with the 16-byte chunks of a row XOR-swizzled by (row / 2) % 4:
// a K-major SW64 wgmma B operand (N = rows, K = the 32 columns).
__host__ __device__ __forceinline__ int item_off(int n, int k) {          // k in [0, 32)
  return (n >> 3) * 512 + (n & 7) * 64 + ((((k >> 3) ^ (n >> 1)) & 3) << 4) + ((k & 7) << 1);
}

// ---------------------------------------------------------------------------------------------
// layout of the tensor-core workspace
// ---------------------------------------------------------------------------------------------
// Forward constants of one network, fp32, in the order the forward kernel's shared-memory copy holds them (float
// offsets): [b_l * S_ACT, l = 0..L-2: 256 each][plain mapping: W0 * S_ACT, [256][3]][output layer: W_{L-1} / S_ACT,
// [out][k_last]][b_{L-1}, out], padded to 16 bytes.
struct FwdConsts { int w0, wl, bl, floats; };
__host__ __device__ constexpr FwdConsts fwd_consts(int L, bool plain, int out, int k_last) {
  const int w0 = (L - 1) * 256, wl = w0 + (plain ? 768 : 0), bl = wl + out * k_last;
  return FwdConsts{w0, wl, bl, (bl + out + 3) / 4 * 4};
}
constexpr int FWD_CST_BYTES = 10752;                 // the largest block: the atlas, 2683 floats

struct NetImages {
  // forward weight items, consumption order: per TC layer, per 64-wide k chunk: hi k 0-31, hi k 32-63, lo k 0-31, lo 32-63
  char* w_fwd; int64_t w_fwd_layer[B200_MAX_LAYERS]; int n_chunks_fwd[B200_MAX_LAYERS];
  float* cst; int cst_floats;             // forward constants (FwdConsts)
  // dgrad weight items (W^T): per layer, per 64-wide chunk of the reduction (out) index: the same four items
  char* w_bwd; int64_t w_bwd_layer[B200_MAX_LAYERS];
  // activation images h_0..h_{L-2} and dZ images: [slot][term][tile][4 atoms][16 KB]
  char* act; char* dz;
  int64_t slot_stride, term_stride;       // bytes
  // 64-wide images: [term][tile][16 KB]: positional encoding (atlas) and the output-layer dZ
  char* pe; char* dzl; int64_t w64_term_stride;
  uint32_t* bits;                         // ReLU flags [slot][rows][8]
  int64_t rows;
};

struct TcLayout { NetImages map, atl; };

static char* align_tc(char* base) { return reinterpret_cast<char*>(round_up(reinterpret_cast<int64_t>(base), 1024)); }
static char* carve_tc(char*& p, int64_t bytes) { char* r = p; p += round_up(bytes, 1024); return r; }

// forward weight images only: all a forward without activation images (the render) needs
static void plan_fwd_weights(const MlpShape& s, TcNet net, char*& p, NetImages* n) {
  const bool pe = tc_pe_first(net);
  int64_t off = 0;
  for (int l = 0; l < s.L; ++l) {
    int chunks = 0;
    const bool tc_layer = pe ? (l <= s.L - 2) : (l >= 1 && l <= s.L - 2);
    if (tc_layer) chunks = (l == 0 ? 0 : HID / 64) + ((l == 0 || s.skip[l]) && pe ? 1 : 0);
    n->n_chunks_fwd[l] = chunks;
    n->w_fwd_layer[l] = off;
    off += (int64_t)chunks * CHUNK_BYTES;
  }
  n->w_fwd = carve_tc(p, off);
  n->cst_floats = fwd_consts(s.L, !pe, s.out_dim, s.K[s.L - 1]).floats;
  n->cst = reinterpret_cast<float*>(carve_tc(p, (int64_t)n->cst_floats * 4));
}

static void plan_net(const MlpShape& s, int64_t rows, TcNet net, char*& p, NetImages* n) {
  const int64_t tiles = rows / TM;
  const bool pe = tc_pe_first(net);
  n->rows = rows;
  plan_fwd_weights(s, net, p, n);
  int64_t off = 0;
  for (int l = 0; l < s.L; ++l) {
    n->w_bwd_layer[l] = off;
    const bool used = l <= s.L - 2 && (pe || l >= 1);
    if (used) off += (int64_t)(HID / 64) * CHUNK_BYTES;
  }
  n->w_bwd = carve_tc(p, off);
  n->term_stride = tiles * TILE_IMG_BYTES;
  n->slot_stride = 2 * n->term_stride;
  n->act = carve_tc(p, (int64_t)(s.L - 1) * n->slot_stride);
  n->dz = carve_tc(p, (int64_t)(s.L - 1) * n->slot_stride);
  n->w64_term_stride = tiles * ATOM_BYTES;
  n->pe = pe ? carve_tc(p, 2 * n->w64_term_stride) : nullptr;
  n->dzl = carve_tc(p, 2 * n->w64_term_stride);
  n->bits = reinterpret_cast<uint32_t*>(carve_tc(p, (int64_t)(s.L - 1) * rows * 32));
}

int64_t tc_plan(const MlpShape& ms, const MlpShape& as, int64_t rows_map, int64_t rows_atlas, char* base,
                TcPlan* out) {
  char* p = align_tc(base);
  TcLayout lay{};
  plan_net(ms, rows_map, tc_net_of(ms), p, &lay.map);
  plan_net(as, rows_atlas, TcNet::Atlas, p, &lay.atl);
  if (out) { out->base = base; out->bytes = p - base; out->rows_map = rows_map; out->rows_atlas = rows_atlas; }
  return p - base;
}

static TcLayout layout_of(const TcStep& s) {
  char* p = align_tc(s.plan->base);
  TcLayout lay{};
  plan_net(*s.ms, s.plan->rows_map, tc_net_of(*s.ms), p, &lay.map);
  plan_net(*s.as, s.plan->rows_atlas, TcNet::Atlas, p, &lay.atl);
  return lay;
}

// ---------------------------------------------------------------------------------------------
// weight preparation
// ---------------------------------------------------------------------------------------------
struct PrepJob {
  const float* W; int ldw;          // fp32 weight [N][ldw]
  int n_rows, k0, k_cnt;            // valid image rows and the window [k0, k0+k_cnt) of the other index
  int transpose;                    // 0: image(row=n, col=k-k0) = W[n][k];  1: image(row=k, col=n-k0) = W[n][k]
  char* hi; char* lo;               // destination: two 16 KB items each (k 0-31, k 32-63), zero padded
  float* f32; float f32_scale;      // non-null: a forward-constant job instead, f32[i] = W[i] * f32_scale, i < n_rows
};
constexpr int MAX_PREP_JOBS = 128;
struct PrepJobs { PrepJob j[MAX_PREP_JOBS]; int n; };

__global__ void tc_prep_kernel(const PrepJobs* __restrict__ jobs_ptr) {
  const PrepJob jb = jobs_ptr->j[blockIdx.x >> 2];
  if (jb.f32) {
    // the same fp32 products the forward kernel formed from the parameters before (no fast math: bit for bit)
    for (int i = (blockIdx.x & 3) * blockDim.x + threadIdx.x; i < jb.n_rows; i += 4 * blockDim.x)
      jb.f32[i] = jb.W[i] * jb.f32_scale;
    return;
  }
  // one job = 256 rows x 64 cols; this block does 64 rows; thread handles one 16-byte chunk at a time
  for (int e = threadIdx.x; e < 64 * 8; e += blockDim.x) {
    const int row = (blockIdx.x & 3) * 64 + (e >> 3), c8 = (e & 7) * 8;
    float v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int col = c8 + q;
      v[q] = 0.f;
      if (row < jb.n_rows && col < jb.k_cnt)
        v[q] = jb.transpose ? jb.W[(int64_t)(jb.k0 + col) * jb.ldw + row] : jb.W[(int64_t)row * jb.ldw + jb.k0 + col];
    }
    uint32_t h[4], l[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) split2_f16(v[2 * q] * S_W, v[2 * q + 1] * S_W, h[q], l[q]);
    const int off = (c8 >> 5) * ITEM_BYTES + item_off(row, c8 & 31);
    *reinterpret_cast<uint4*>(jb.hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(jb.lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

// ---------------------------------------------------------------------------------------------
// shared pieces of the fused kernels
// ---------------------------------------------------------------------------------------------
template <int NST>
struct Pipe {                        // weight-image ring shared by the producer warp and the consumer warpgroups
  uint64_t* full; uint64_t* empty; char* stage;
  uint32_t it;                       // running item counter
  __device__ __forceinline__ int slot() const { return it % NST; }
  __device__ __forceinline__ uint32_t parity() const { return (it / NST) & 1; }
};

struct TileIter {                    // static round-robin over the live tiles of a group-major batch
  int t0, tf, tb, total, cap_tiles, n_groups, gf, gb;
  // counters: [0] rows of an ordinary group, [5] / [6] rows of the compacted flow-match groups g_fwd / g_bwd (-1: the
  // batch has no such group); nullptr: every row of every group is live
  __device__ __forceinline__ void init(int cap, int groups, const int* counters, int g_fwd, int g_bwd) {
    cap_tiles = cap / TM;
    n_groups = groups;
    gf = (counters && g_fwd < groups) ? g_fwd : -1;
    gb = (counters && g_bwd < groups) ? g_bwd : -1;
    t0 = counters ? min(cap_tiles, (counters[0] + TM - 1) / TM) : cap_tiles;
    tf = gf >= 0 ? min(cap_tiles, (counters[5] + TM - 1) / TM) : t0;
    tb = gb >= 0 ? min(cap_tiles, (counters[6] + TM - 1) / TM) : t0;
    total = t0 * (groups - (gf >= 0) - (gb >= 0)) + (gf >= 0 ? tf : 0) + (gb >= 0 ? tb : 0);
  }
  __device__ __forceinline__ int group_tiles(int g) const { return g == gf ? tf : (g == gb ? tb : t0); }
  __device__ __forceinline__ int global_tile(int t) const {
    for (int g = 0; g < n_groups; ++g) {
      const int n = group_tiles(g);
      if (t < n) return g * cap_tiles + t;
      t -= n;
    }
    return 0;
  }
};

// n_items consecutive weight items into the ring; `bytes` < ITEM_BYTES sends only the first rows of each (the n64 dPE
// product reads 64 of the 256 rows)
template <int NST>
__device__ __forceinline__ void produce_items(Pipe<NST>& pp, const char* src, int n_items, uint32_t bytes = ITEM_BYTES) {
  for (int i = 0; i < n_items; ++i) {
    mbar_wait(&pp.empty[pp.slot()], pp.parity() ^ 1);
    mbar_expect_tx(&pp.full[pp.slot()], bytes);
    bulk_g2s(pp.stage + pp.slot() * ITEM_BYTES, src + (int64_t)i * ITEM_BYTES, bytes, &pp.full[pp.slot()]);
    ++pp.it;
  }
}

// Thread geometry of the fused kernels: warps 0..7 are two consumer warpgroups, each owning 64 rows of the 128-row tile
// (its A operand rows, its wgmma accumulator rows); warps 8..11 are the producer warpgroup (one lane streams the weight
// images).  Registers are allotted per warpgroup: the producer gives most of its share to the consumers.
constexpr int CONSUMER_WGS = 2;
constexpr int CONSUMERS = CONSUMER_WGS * 128;
constexpr int TC_THREADS = CONSUMERS + 128;
constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 224;      // 128 * 56 + 256 * 224 <= 64 K
constexpr int EMPTY_ARRIVALS = CONSUMER_WGS * 4;      // one per consumer warp
constexpr int WG_ROW_BYTES = 8192;                    // a warpgroup's 64 rows inside one 64-column atom block

struct Consumer {
  int g, w4, lane, q, tid;       // warpgroup, warp in the group, lane, lane % 4, thread index in the group
  int m0;                        // first of this thread's two tile rows (m0, m0 + 8)
  bool warp_leader, leader;      // lane 0 of the warp / thread 0 of the warpgroup
  __device__ __forceinline__ void init() {
    const int warp = warp_uniform();
    lane = threadIdx.x & 31; q = lane & 3;
    g = warp >> 2; w4 = warp & 3;
    tid = threadIdx.x & 127;
    m0 = 64 * g + 16 * w4 + (lane >> 2);
    warp_leader = lane == 0;
    leader = tid == 0;
  }
  __device__ __forceinline__ void sync() const { named_bar(1 + g, 128); }
};

// A operand tile in shared memory: [term][4 atom blocks of 64 columns][128 rows x 128 B], i.e. exactly the byte layout
// of one tile of an activation / dZ image, so it doubles as the staging buffer of the image's bulk store
__host__ __device__ __forceinline__ int tile_off(int m, int col) { return (col >> 6) * ATOM_BYTES + atom_off(m, col & 63); }

// One 16 KB weight item (B: 256 rows x 32 k, K-major SW64) against 32 columns of this warpgroup's rows of the A tile
// (a_hi / a_lo: their first column inside a 64-column atom block): D += A_hi * B (+ A_lo * B when with_lo), one k16
// step after the other.  The item read before this one is released once its MMAs have completed.
template <int NST, int NN>
__device__ __forceinline__ void consume_item(Pipe<NST>& pp, float (&acc)[NN / 2], uint32_t a_hi, uint32_t a_lo, bool with_lo,
                                             uint32_t& scale, int& pending, const Consumer& c) {
  mbar_wait(&pp.full[pp.slot()], pp.parity());
  const uint32_t sb = smem_u32(pp.stage + pp.slot() * ITEM_BYTES);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    const uint64_t bd = make_desc_sw64(sb + ks * 32, 512);
    if constexpr (NN == 256) wgmma_n256<0, 0>(*reinterpret_cast<float(*)[128]>(&acc), make_desc(a_hi + ks * 32, 16, 1024), bd, scale);
    else wgmma_n64<0, 0>(*reinterpret_cast<float(*)[32]>(&acc), make_desc(a_hi + ks * 32, 16, 1024), bd, scale);
    scale = 1u;
    if (with_lo) {
      if constexpr (NN == 256) wgmma_n256<0, 0>(*reinterpret_cast<float(*)[128]>(&acc), make_desc(a_lo + ks * 32, 16, 1024), bd, 1u);
      else wgmma_n64<0, 0>(*reinterpret_cast<float(*)[32]>(&acc), make_desc(a_lo + ks * 32, 16, 1024), bd, 1u);
    }
  }
  wgmma_commit();
  wgmma_wait<1>();
  if (pending >= 0 && c.warp_leader) mbar_arrive(&pp.empty[pending]);
  pending = pp.slot();
  ++pp.it;
}
// MMAs of one 64-wide k chunk, per k16 step:  D += A_hi*B_hi + A_lo*B_hi  (two B_hi items)  then  D += A_hi*B_lo  (two
// B_lo items); 64 bytes of an A row are 32 columns
template <int NST, int NN>
__device__ __forceinline__ void consume_chunk(Pipe<NST>& pp, float (&acc)[NN / 2], uint32_t a_hi, uint32_t a_lo,
                                              uint32_t& scale, int& pending, const Consumer& c) {
  consume_item<NST, NN>(pp, acc, a_hi, a_lo, true, scale, pending, c);
  consume_item<NST, NN>(pp, acc, a_hi + 64, a_lo + 64, true, scale, pending, c);
  consume_item<NST, NN>(pp, acc, a_hi, a_lo, false, scale, pending, c);
  consume_item<NST, NN>(pp, acc, a_hi + 64, a_lo + 64, false, scale, pending, c);
}
template <int NST, int R>
__device__ __forceinline__ void finish_pass(Pipe<NST>& pp, float (&acc)[R], int& pending, const Consumer& c) {
  wgmma_wait<0>();
  acc_fence(acc);
  if (pending >= 0 && c.warp_leader) mbar_arrive(&pp.empty[pending]);
  pending = -1;
}

// this warpgroup's rows of the A tile -> the tile of an HBM image (both terms), one bulk store per atom block and term
__device__ __forceinline__ void store_tile_rows(const Consumer& c, const char* a_tile, char* g_img, int64_t term_stride) {
  if (!c.leader) return;
#pragma unroll
  for (int term = 0; term < 2; ++term)
#pragma unroll
    for (int j = 0; j < 4; ++j)
      bulk_s2g(g_img + term * term_stride + j * ATOM_BYTES + c.g * WG_ROW_BYTES,
               a_tile + term * TILE_IMG_BYTES + j * ATOM_BYTES + c.g * WG_ROW_BYTES, WG_ROW_BYTES);
  bulk_commit();
}
// before the A tile is overwritten: every MMA of the warpgroup has completed (finish_pass) and the bulk store of the
// previous contents has read them
__device__ __forceinline__ void a_tile_reusable(const Consumer& c) {
  if (c.leader) bulk_wait_read0();
  c.sync();
}
// after the A tile was written with generic stores: visible to the next MMAs (async proxy) and to the bulk store
__device__ __forceinline__ void a_tile_written(const Consumer& c) {
  fence_proxy_async_smem();
  c.sync();
}

__device__ __forceinline__ uint32_t relu_flag(float v) { return (uint32_t)(-(int)__float_as_uint(v)) >> 31; }   // v > +0

// ReLU flags of this thread's pair of columns (col, col+1) in its 16-column piece, OR-ed over the quad -> 16-bit word
// (flag of column i of the piece at bit 15 - i); lane q == 0 of the quad stores it
__device__ __forceinline__ uint32_t piece_bits(uint32_t f0, uint32_t f1, int col) {
  const int i = col & 15;
  uint32_t b = (f0 << (15 - i)) | (f1 << (14 - i));
  return b;
}
__device__ __forceinline__ uint32_t quad_or(uint32_t b) {
  b |= __shfl_xor_sync(0xffffffffu, b, 1);
  b |= __shfl_xor_sync(0xffffffffu, b, 2);
  return b;
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// dynamic shared memory map: [A tile hi 64 KB | lo 64 KB][weight ring][aux tile 32 KB (atlas forward)][consts][barriers]
constexpr int SMEM_A = 2 * TILE_IMG_BYTES;
constexpr int SMEM_AUX = 2 * ATOM_BYTES;
// backward: per consumer warpgroup the B operand of the row-sum MMAs (64 rows x 8 fp16) and a slice of gradient
// accumulators (bias gradients of layers 0..L-2, + dW0 of the mapping: 7 * 256 for the atlas, 5 * 256 + 768 for the
// 6-layer mapping)
constexpr int RSUM_B_BYTES = 64 * 16;
constexpr int BWD_ACC_FLOATS = 5 * 256 + 768;
constexpr int SMEM_BWD_CONST_FLOATS = CONSUMER_WGS * (RSUM_B_BYTES / 4 + BWD_ACC_FLOATS);
constexpr int SMEM_BARS = 256;
constexpr int SMEM_MAX = 227 * 1024;                         // opt-in shared memory of one sm_90 CTA
// Every kernel keeps as many 16 KB weight slots as the shared memory allows next to the A tile and its constants.  The
// forward kernels hold their network's forward constants (FwdConsts, <= 10.5 KB) resident, which costs one slot: 5 in
// the mapping forward, 3 in the atlas forward, which also holds the positional-encoding tile.  The backward kernels
// hold their gradient accumulators and row-sum operands (5 slots).
template <bool ATLAS, bool BWD> struct KCfg {
  static constexpr int NST = BWD ? 5 : (ATLAS ? 3 : 5);
  static constexpr int SMEM = SMEM_A + NST * ITEM_BYTES + (ATLAS && !BWD ? SMEM_AUX : 0) +
                              (BWD ? SMEM_BWD_CONST_FLOATS * 4 : FWD_CST_BYTES) + SMEM_BARS;
  static_assert(SMEM <= SMEM_MAX, "fused kernel exceeds the shared memory of one CTA");
  static_assert(SMEM + ITEM_BYTES > SMEM_MAX, "one more weight slot would fit");
  static_assert(2 * NST * 8 + 8 <= SMEM_BARS, "ring and constant barriers exceed their shared-memory slot");
};

template <int NST>
struct SmemMap {
  char* a_tile; char* stage; char* aux; float* cst;
  uint64_t* full; uint64_t* empty;   // [NST] each; the forward's constants barrier follows at empty[NST]
  __device__ __forceinline__ void init(char* raw, int aux_bytes, int cst_floats) {
    char* p = raw;                                   // 1024-aligned (checked in setup_cta)
    a_tile = p; p += SMEM_A;
    stage = p; p += NST * ITEM_BYTES;
    aux = p; p += aux_bytes;
    cst = reinterpret_cast<float*>(p); p += cst_floats * 4;
    full = reinterpret_cast<uint64_t*>(p);
    empty = full + NST;
  }
};

template <int NST>
__device__ __forceinline__ void setup_cta(SmemMap<NST>& sm, bool cst_bar = false) {
  if (threadIdx.x == 0) {
    if (smem_u32(sm.a_tile) & 1023u) __trap();   // the swizzled operand layouts need 1024-byte alignment
    for (int i = 0; i < NST; ++i) { mbar_init(&sm.full[i], 1); mbar_init(&sm.empty[i], EMPTY_ARRIVALS); }
    if (cst_bar) mbar_init(&sm.empty[NST], 1);
    fence_barrier_init();
  }
  __syncthreads();
}
constexpr int BAR_CONSUMERS = 9;                         // named barrier of all consumer threads

struct FwdParams {
  const float* x;            // mapping: [rows][4] (x, y, t, 0);  atlas: uv [rows][2]
  float* y;                  // mapping: uv [rows][2];  atlas: y [rows][3]
  const float* params;       // fp32 parameters of this network
  int64_t w_off[B200_MAX_LAYERS], b_off[B200_MAX_LAYERS];
  NetImages img;
  int cap, n_groups; const int* n_valid;
  int g_fwd, g_bwd;          // groups compacted to counters[5] / counters[6] rows (-1: none; see TileIter)
  float in_scale, in_shift;  // atlas: network input = x * in_scale + in_shift (0.5, 0.5 inside the loop: uv -> [0,1])
  int store_images;          // 0: inference (render / IMLP.forward without grad): no activation images, no flags
  int tanh_out;
  int pe_freqs;              // 3-input PE-first networks: frequencies of the encoding (1..10, 6 columns each)
};

// =============================================================================================
// forward
// =============================================================================================
// One 128-row tile walks through all layers on chip.  Per layer each consumer warpgroup runs the MMAs of its 64 rows
// (A tile in shared memory, weight items from the ring), then its epilogue turns the accumulator registers into the next
// layer's A operand (bias + ReLU + flag bits + 2-term split) in place and bulk-stores those rows to the activation image.
// ATLAS = true: the positional encoding feeds layer 0, which runs on the tensor cores.  VAR = 0: the atlas network (2
// inputs, 10 frequencies, skips at 4 and 7, 3 outputs).  VAR > 0: the 3-input family (3 inputs, P.pe_freqs frequencies
// in one 64-column chunk, no skips, VAR outputs, no input gradient): the alpha network of the segmentation variant
// (NL = 8, VAR = 1, 5 frequencies) and the position-encoded mappings (NL = 6 or 4, VAR = 2).
template <bool ATLAS, int NL = (ATLAS ? 8 : 6), int VAR = 0>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_fwd_kernel(const __grid_constant__ FwdParams P) {
  extern __shared__ __align__(1024) char smem_raw[];
  constexpr int NST = KCfg<ATLAS, false>::NST;
  SmemMap<NST> sm; sm.init(smem_raw, ATLAS ? SMEM_AUX : 0, FWD_CST_BYTES / 4);
  const int warp = warp_uniform(), lane = threadIdx.x & 31;
  constexpr int L = NL;                                   // mapping-shaped networks: 6 (stage-1 script) or 4 layers
  constexpr int FIRST_TC = ATLAS ? 0 : 1;
  constexpr int LAST_TC = L - 2;
  constexpr bool PE3 = ATLAS && VAR > 0;                  // the 3-input family
  constexpr bool SKIPS = ATLAS && !PE3;                   // PE chunk concatenated at layers 4 and L-1
  constexpr int OUT = ATLAS ? (PE3 ? VAR : 3) : 2;
  constexpr int KLAST = SKIPS ? 296 : 256;
  constexpr FwdConsts CST = fwd_consts(L, !ATLAS, OUT, KLAST);
  static_assert(CST.floats * 4 <= FWD_CST_BYTES, "forward constants exceed their shared-memory slot");
  uint64_t* cst_full = &sm.empty[NST];
  // real encoding columns of the 3-input family; the alpha network's 5 frequencies are part of its identity (tc_net_of)
  const int pe_cols = VAR == 1 ? 30 : 6 * P.pe_freqs;
  setup_cta(sm, true);
  TileIter ti; ti.init(P.cap, P.n_groups, P.n_valid, P.g_fwd, P.g_bwd);

  if (warp >= CONSUMER_WGS * 4) {
    // ------------------------------------------------------------------ producer (consumption order)
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == CONSUMER_WGS * 4 && lane == 0) {
      // the constants, once per CTA, ahead of the first weight item
      mbar_expect_tx(cst_full, CST.floats * 4);
      bulk_g2s(sm.cst, P.img.cst, CST.floats * 4, cst_full);
      Pipe<NST> pp{sm.full, sm.empty, sm.stage, 0};
      for (int t = blockIdx.x; t < ti.total; t += gridDim.x)
        for (int l = FIRST_TC; l <= LAST_TC; ++l) {
          const char* base = P.img.w_fwd + P.img.w_fwd_layer[l];
          if (ATLAS && l == 0) { produce_items(pp, base, 4); continue; }
          if (SKIPS && l == 4) produce_items(pp, base + (int64_t)4 * CHUNK_BYTES, 4);      // skip (PE) chunk first
          produce_items(pp, base, 16);
        }
    }
    return;
  }
  // ------------------------------------------------------------------ consumer warpgroups
  setmaxnreg_inc<CONSUMER_REGS>();
  Consumer c; c.init();
  Pipe<NST> pp{sm.full, sm.empty, sm.stage, 0};
  int pending = -1;
  const float inv_scale = 1.0f / S_W;                   // D / (S_a S_w) * S_a : activations stay scaled by S_ACT
  const float* wlast = sm.cst + CST.wl;                 // W_{L-1} / S_ACT
  const uint32_t a_rows = smem_u32(sm.a_tile) + c.g * WG_ROW_BYTES;
  const uint32_t aux_rows = smem_u32(sm.aux) + c.g * WG_ROW_BYTES;
  float acc[128];
  mbar_wait(cst_full, 0);
  for (int t = blockIdx.x; t < ti.total; t += gridDim.x) {
    const int gt = ti.global_tile(t);
    const int64_t row0 = (int64_t)gt * TM + c.m0;
    uint16_t* bits_row = reinterpret_cast<uint16_t*>(P.img.bits) + row0 * 16;   // flags of row0 in slot 0
    // epilogue store of one column pair of one row: split into the A tile
    auto put = [&](int m, int col, float v0, float v1) {
      uint32_t h, lo;
      split2_packed(v0, v1, h, lo);
      const int off = tile_off(m, col);
      *reinterpret_cast<uint32_t*>(sm.a_tile + off) = h;
      *reinterpret_cast<uint32_t*>(sm.a_tile + TILE_IMG_BYTES + off) = lo;
    };
    // flags of the two 8-column groups of a 16-column piece: the even group is held, the odd one completes the word
    uint32_t held0 = 0, held1 = 0;
    auto flags_out = [&](int slot, int i, int col, uint32_t b0, uint32_t b1) {
      if ((i & 1) == 0) { held0 = b0; held1 = b1; return; }
      b0 = quad_or(b0 | held0); b1 = quad_or(b1 | held1);
      if (P.store_images && c.q == 0) {
        uint16_t* dst = bits_row + (int64_t)slot * P.img.rows * 16 + (col >> 4);
        dst[0] = (uint16_t)b0;
        dst[8 * 16] = (uint16_t)b1;
      }
    };
    // one bias + ReLU column pair of a tensor-core layer's accumulators: v = relu(acc / S_W + b * S_ACT)
    auto bias_relu = [&](const float* bias, int i, int col, float (&v)[4]) {
      const float2 bs = *reinterpret_cast<const float2*>(bias + col);
      v[0] = fmaxf(__fmaf_rn(acc[4 * i], inv_scale, bs.x), 0.f);
      v[1] = fmaxf(__fmaf_rn(acc[4 * i + 1], inv_scale, bs.y), 0.f);
      v[2] = fmaxf(__fmaf_rn(acc[4 * i + 2], inv_scale, bs.x), 0.f);
      v[3] = fmaxf(__fmaf_rn(acc[4 * i + 3], inv_scale, bs.y), 0.f);
    };
    // ---------------- prologue: layer-0 input
    if (ATLAS) {
      // positional encoding of in = x*in_scale+in_shift (implicit_neural_networks.py:9-13) into the aux tile
      // (K-major SW128, columns k*4 + {sin x0, sin x1, cos x0, cos x1}); 8-column chunks of this warpgroup's rows
      c.sync();                                          // previous tile's readers of the aux rows are done
      for (int task = c.tid; task < 64 * 8; task += 128) {
        const int m = 64 * c.g + (task & 63), c8 = task >> 6;
        const int64_t row = (int64_t)gt * TM + m;
        float in[3] = {0.f, 0.f, 0.f};
        if (PE3) {                                       // rows padded to 4 floats, like the mapping's
          const float4 xv = *reinterpret_cast<const float4*>(P.x + row * 4);
          in[0] = xv.x * P.in_scale + P.in_shift; in[1] = xv.y * P.in_scale + P.in_shift; in[2] = xv.z * P.in_scale + P.in_shift;
        } else {
          const float2 uv = *reinterpret_cast<const float2*>(P.x + row * 2);
          in[0] = uv.x * P.in_scale + P.in_shift; in[1] = uv.y * P.in_scale + P.in_shift;
        }
        float vals[8];
        if (PE3) {
          // column c = k*6 + r: r < 3 -> sin(x_r b_k), else cos(x_{r-3} b_k); pe_cols real columns
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int cc = c8 * 8 + i;
            float v = 0.f;
            if (cc < pe_cols) {
              const int k = cc / 6, r = cc - k * 6;
              const float a = in[r < 3 ? r : r - 3] * pe_freq(k);
              v = r < 3 ? sinf(a) : cosf(a);
            }
            vals[i] = v * S_ACT;
          }
        } else {
#pragma unroll
          for (int half_k = 0; half_k < 2; ++half_k) {
            const int k = c8 * 2 + half_k;
            float s0 = 0.f, s1 = 0.f, c0 = 0.f, c1 = 0.f;
            if (k < 10) {
              const float bk = pe_freq(k);
              const float a0 = in[0] * bk, a1 = in[1] * bk;
              s0 = sinf(a0); s1 = sinf(a1); c0 = cosf(a0); c1 = cosf(a1);
            }
            vals[half_k * 4 + 0] = s0 * S_ACT; vals[half_k * 4 + 1] = s1 * S_ACT;
            vals[half_k * 4 + 2] = c0 * S_ACT; vals[half_k * 4 + 3] = c1 * S_ACT;
          }
        }
        uint32_t h[4], lo[4];
#pragma unroll
        for (int q2 = 0; q2 < 4; ++q2) split2_f16(vals[2 * q2], vals[2 * q2 + 1], h[q2], lo[q2]);
        const int off = atom_off(m, c8 * 8);
        const uint4 vh = make_uint4(h[0], h[1], h[2], h[3]), vl = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        *reinterpret_cast<uint4*>(sm.aux + off) = vh;
        *reinterpret_cast<uint4*>(sm.aux + ATOM_BYTES + off) = vl;
        if (P.store_images) {
          char* g_hi = P.img.pe + (int64_t)gt * ATOM_BYTES;
          *reinterpret_cast<uint4*>(g_hi + off) = vh;
          *reinterpret_cast<uint4*>(g_hi + P.img.w64_term_stride + off) = vl;
        }
      }
      fence_proxy_async_smem();                          // generic-proxy smem writes -> visible to the MMAs
      c.sync();
    } else {
      // layer 0 (3 -> 256) on CUDA cores: h0 = relu(W0 x + b0)
      const float4 x0 = *reinterpret_cast<const float4*>(P.x + row0 * 4);
      const float4 x1 = *reinterpret_cast<const float4*>(P.x + (row0 + 8) * 4);
      const float* b0s = sm.cst;                         // b0 * S_ACT
      const float* w0s = sm.cst + CST.w0;                // W0 * S_ACT, [256][3]
      a_tile_reusable(c);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = 8 * i + 2 * c.q;
        const float2 bs = *reinterpret_cast<const float2*>(b0s + col);
        const float2 wa = *reinterpret_cast<const float2*>(w0s + col * 3);      // W0[col][0..1]
        const float2 wb = *reinterpret_cast<const float2*>(w0s + col * 3 + 2);  // W0[col][2], W0[col+1][0]
        const float2 wc = *reinterpret_cast<const float2*>(w0s + col * 3 + 4);  // W0[col+1][1..2]
        const float w[2][3] = {{wa.x, wa.y, wb.x}, {wb.y, wc.x, wc.y}}, b[2] = {bs.x, bs.y};
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          acc[4 * i + e] = fmaxf(__fmaf_rn(x0.z, w[e][2], __fmaf_rn(x0.y, w[e][1], __fmaf_rn(x0.x, w[e][0], b[e]))), 0.f);
          acc[4 * i + 2 + e] = fmaxf(__fmaf_rn(x1.z, w[e][2], __fmaf_rn(x1.y, w[e][1], __fmaf_rn(x1.x, w[e][0], b[e]))), 0.f);
        }
        put(c.m0, col, acc[4 * i], acc[4 * i + 1]);
        put(c.m0 + 8, col, acc[4 * i + 2], acc[4 * i + 3]);
        flags_out(0, i, col, piece_bits(relu_flag(acc[4 * i]), relu_flag(acc[4 * i + 1]), col),
                  piece_bits(relu_flag(acc[4 * i + 2]), relu_flag(acc[4 * i + 3]), col));
      }
      a_tile_written(c);
      if (P.store_images) store_tile_rows(c, sm.a_tile, P.img.act + (int64_t)gt * TILE_IMG_BYTES, P.img.term_stride);
    }
    // ---------------- tensor-core layers
    auto mma_layer = [&](int l) {
      uint32_t scale = 0u;
      if (ATLAS && (l == 0 || (SKIPS && l == 4)))
        consume_chunk<NST, 256>(pp, acc, aux_rows, aux_rows + ATOM_BYTES, scale, pending, c);
      if (l > 0)
        for (int kc = 0; kc < 4; ++kc)
          consume_chunk<NST, 256>(pp, acc, a_rows + kc * ATOM_BYTES, a_rows + TILE_IMG_BYTES + kc * ATOM_BYTES, scale,
                                  pending, c);
      finish_pass(pp, acc, pending, c);
    };
    // every tensor-core layer: bias + ReLU + flags + split into the A tile (the next layer's operand, or the last
    // layer's activation image); the last one also feeds the output layer on CUDA cores
    float outacc[2][OUT];
#pragma unroll
    for (int jj = 0; jj < OUT; ++jj) outacc[0][jj] = outacc[1][jj] = 0.f;
#pragma unroll 1
    for (int l = FIRST_TC; l <= LAST_TC; ++l) {
      mma_layer(l);
      const bool last = l == LAST_TC;
      const float* bias = sm.cst + l * 256;
      a_tile_reusable(c);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = 8 * i + 2 * c.q;
        float v[4];
        bias_relu(bias, i, col, v);
        if (last) {
#pragma unroll
          for (int jj = 0; jj < OUT; ++jj) {
            const float2 w = *reinterpret_cast<const float2*>(wlast + jj * KLAST + col);
            outacc[0][jj] = fmaf(v[1], w.y, fmaf(v[0], w.x, outacc[0][jj]));
            outacc[1][jj] = fmaf(v[3], w.y, fmaf(v[2], w.x, outacc[1][jj]));
          }
        }
        if (!last || P.store_images) {
          put(c.m0, col, v[0], v[1]);
          put(c.m0 + 8, col, v[2], v[3]);
        }
        flags_out(l, i, col, piece_bits(relu_flag(v[0]), relu_flag(v[1]), col),
                  piece_bits(relu_flag(v[2]), relu_flag(v[3]), col));
      }
      a_tile_written(c);
      if (P.store_images)
        store_tile_rows(c, sm.a_tile, P.img.act + (int64_t)l * P.img.slot_stride + (int64_t)gt * TILE_IMG_BYTES,
                        P.img.term_stride);
    }
    // ---------------- output layer (+ skip part for the atlas) and tanh; the four lanes of a quad share the rows
    if (SKIPS) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = c.m0 + 8 * rr;
        for (int k = c.q * 10; k < c.q * 10 + 10; ++k) {
          const int off = atom_off(m, k);
          const float pv = __half2float(*reinterpret_cast<const __half*>(sm.aux + off)) +
                           __half2float(*reinterpret_cast<const __half*>(sm.aux + ATOM_BYTES + off));     // S_ACT * pe
#pragma unroll
          for (int jj = 0; jj < OUT; ++jj)
            outacc[rr][jj] = fmaf(pv, wlast[jj * KLAST + 256 + k], outacc[rr][jj]);
        }
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
      for (int jj = 0; jj < OUT; ++jj) {
        const float o = quad_sum(outacc[rr][jj]) + sm.cst[CST.bl + jj];
        if (c.q == 0) P.y[(row0 + 8 * rr) * OUT + jj] = P.tanh_out ? tanhf(o) : o;
      }
  }
  if (c.leader) bulk_wait_all0();
}

// =============================================================================================
// backward (dgrad chain + first-layer / bias gradients; the 64-wide output-layer dZ image)
// =============================================================================================
struct BwdParams {
  const float* dy;           // mapping: d_uv [rows][2];  atlas: d_y [rows][3]
  const float* y;            // network output (tanh applied)
  const float* x;            // mapping: x_map [rows][4]
  float* d_in;               // atlas: d_uv [rows][2] (accumulated: += 0.5 * dPE/din)
  const float* params;       // fp32 parameters of this network
  float* grads;              // fp32 gradient block of this network
  int64_t w_off[B200_MAX_LAYERS], b_off[B200_MAX_LAYERS];
  NetImages img;
  int cap, n_groups; const int* n_valid;
  int* gmax_bits;            // [0] max |dL/dy| from the loss head, [1] max |dL/duv| after the atlas backward
  int g_fwd, g_bwd;
  float in_scale;            // atlas: d(network input)/d(x) (0.5 inside the loop)
  int d_in_accumulate;       // atlas: 1 = d_in already holds the direct loss-head gradient (the loop), 0 = overwrite
  int tanh_out;
};

// gmax_bits[0]: max |dL/drgb| (atlas network);  gmax_bits[1]: max |dL/duv| (mapping network: loss head,
// then raised by the atlas backward, whose positional encoding multiplies gradients by up to 2^9*pi).
__device__ __forceinline__ void grad_scales(const int* gmax_bits, bool mapping, float& s_g, float& inv_sg) {
  const float mx = __int_as_float(gmax_bits[mapping ? 1 : 0]);
  int e = 0;
  if (mx > 0.f && mx < 3.0e38f) frexpf(mx, &e);        // mx < 2^e
  e = max(-60, min(60, e));
  s_g = ldexpf(1.0f, 13 - e);                           // mx * s_g < 8192: 8x headroom below the fp16 range
  inv_sg = ldexpf(1.0f, e - 13);                        // (conversions saturate), small entries keep their lo term
}

template <bool ATLAS, int NL = (ATLAS ? 8 : 6), int VAR = 0>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_bwd_kernel(const __grid_constant__ BwdParams P) {
  extern __shared__ __align__(1024) char smem_raw[];
  constexpr int NST = KCfg<ATLAS, true>::NST;
  SmemMap<NST> sm; sm.init(smem_raw, 0, SMEM_BWD_CONST_FLOATS);
  const int warp = warp_uniform(), lane = threadIdx.x & 31;
  constexpr int L = NL;                                   // mapping-shaped networks: 6 (stage-1 script) or 4 layers
  constexpr bool PE3 = ATLAS && VAR > 0;                  // the 3-input family (see tc_fwd_kernel)
  constexpr bool SKIPS = ATLAS && !PE3;                   // PE chunk concatenated at layers 4 and L-1
  constexpr int OUT = ATLAS ? (PE3 ? VAR : 3) : 2;
  constexpr int KLAST = SKIPS ? 296 : 256;
  constexpr int LOW = 1;                                  // dgrad layers L-2 .. 1 (atlas: + the dPE product)
  constexpr bool HAS_DPE = ATLAS && !PE3;                 // input gradient through the positional encoding
  constexpr bool MAPPING = OUT == 2;                      // the 3 -> 2 mappings, with or without encoding
  // per consumer warpgroup: the B operand of its row-sum MMAs and its slice of the gradient accumulators, [bias
  // gradients of layers 0..L-2 (256 each) | (plain mapping) dW0 [256][3]]
  static_assert((L - 1) * 256 + (ATLAS ? 0 : 768) <= BWD_ACC_FLOATS, "gradient accumulators exceed their slice");
  char* rsum_b = reinterpret_cast<char*>(sm.cst);
  float* s_acc = sm.cst + CONSUMER_WGS * RSUM_B_BYTES / 4;
  for (int i = threadIdx.x; i < CONSUMER_WGS * BWD_ACC_FLOATS; i += blockDim.x) s_acc[i] = 0.f;
  setup_cta(sm);
  TileIter ti; ti.init(P.cap, P.n_groups, P.n_valid, P.g_fwd, P.g_bwd);
  float s_g, inv_sg;
  grad_scales(P.gmax_bits, MAPPING, s_g, inv_sg);

  if (warp >= CONSUMER_WGS * 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == CONSUMER_WGS * 4 && lane == 0) {
      Pipe<NST> pp{sm.full, sm.empty, sm.stage, 0};
      for (int t = blockIdx.x; t < ti.total; t += gridDim.x)
        for (int l = L - 2; l >= (HAS_DPE ? 0 : LOW); --l)
          produce_items(pp, P.img.w_bwd + P.img.w_bwd_layer[l], 16, l == 0 ? 64 * 64 : ITEM_BYTES);   // dPE: 64 rows
    }
    return;
  }
  setmaxnreg_inc<CONSUMER_REGS>();
  Consumer c; c.init();
  Pipe<NST> pp{sm.full, sm.empty, sm.stage, 0};
  int pending = -1;
  const float inv_dgrad = inv_sg * (1.0f / S_W);          // D = (S_g dZ)(S_w W)
  const uint16_t* bits16 = reinterpret_cast<const uint16_t*>(P.img.bits);
  const float* wlast = P.params + P.w_off[L - 1];
  const uint32_t a_rows = smem_u32(sm.a_tile) + c.g * WG_ROW_BYTES;
  const uint32_t b_rows = smem_u32(rsum_b) + c.g * RSUM_B_BYTES;
  float* g_acc = s_acc + c.g * BWD_ACC_FLOATS;
  float acc[128];
  // Sums over this warpgroup's 64 rows of the dZ tile it has just written (both terms), on the tensor cores:
  // D[n][j] = sum_m dZ[m][n] B[m][j], A = the tile as an MN-major operand (M = its 256 columns, one atom block per
  // m64n8k16, K = the rows), B = [1, 0, x_hi, x_lo, y_hi, y_lo, t_hi, t_lo] per row (S_ACT * x; plain mapping, else
  // [1, 0, ...]).  Lane q of a quad holds B columns 2q, 2q + 1, one hi / lo pair: q = 0 the bias gradient of layer
  // `slot`, q = 1..3 (the plain mapping's slot 0) dW0[n][q - 1].  Every element of the slice has one owning thread: plain
  // loads and stores.  The accumulator is the first 16 registers of acc, free once the epilogue has written the tile.
  auto row_sums = [&](int slot) {
    float (&red)[16] = *reinterpret_cast<float(*)[16]>(&acc);
    // two base descriptors, built here and not hoisted out of the tile loop (36 live descriptors would spill);
    // the others add the byte offset / 16 to the start-address field
    uint32_t a_base = a_rows, b_base = b_rows;
    asm volatile("" : "+r"(a_base), "+r"(b_base));
    const uint64_t ad = make_desc(a_base, ATOM_BYTES, 1024), bd = make_desc_rows16(b_base);
    wgmma_fence();
#pragma unroll
    for (int blk = 0; blk < 4; ++blk)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {                   // 16 rows = two groups of 8 rows
        const uint64_t a = ad + ((blk * ATOM_BYTES + ks * 2048) >> 4), b = bd + ((ks * 256) >> 4);
        float (&d)[4] = *reinterpret_cast<float(*)[4]>(&red[4 * blk]);
        wgmma_n8<1, 1>(d, a, b, ks > 0 ? 1u : 0u);
        wgmma_n8<1, 1>(d, a + (TILE_IMG_BYTES >> 4), b, 1u);
      }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(red);
    const bool w0 = !ATLAS && slot == 0;
    if (c.q == 0 || w0) {
#pragma unroll
      for (int blk = 0; blk < 4; ++blk)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int n = 64 * blk + 16 * c.w4 + (c.lane >> 2) + 8 * rr;
          const float v = (red[4 * blk + 2 * rr] + red[4 * blk + 2 * rr + 1]) * inv_sg;
          if (c.q == 0) g_acc[slot * 256 + n] += v;
          else g_acc[(L - 1) * 256 + n * 3 + c.q - 1] += v * (1.0f / S_ACT);
        }
    }
  };
  auto put = [&](int m, int col, float v0, float v1) {
    uint32_t h, lo;
    split2_packed(__fmul_rn(v0, s_g), __fmul_rn(v1, s_g), h, lo);
    const int off = tile_off(m, col);
    *reinterpret_cast<uint32_t*>(sm.a_tile + off) = h;
    *reinterpret_cast<uint32_t*>(sm.a_tile + TILE_IMG_BYTES + off) = lo;
  };
  for (int t = blockIdx.x; t < ti.total; t += gridDim.x) {
    const int gt = ti.global_tile(t);
    const int64_t row0 = (int64_t)gt * TM + c.m0;
    // ---------------- output layer: tanh', bias gradient, the 64-wide dZ_L image, dA_{L-1}
    float dzl[2][OUT];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
      for (int jj = 0; jj < OUT; ++jj) {
        const int64_t row = row0 + 8 * rr;
        const float yv = P.y[row * OUT + jj];
        dzl[rr][jj] = P.dy[row * OUT + jj] * (P.tanh_out ? (1.0f - yv * yv) : 1.0f);
      }
#pragma unroll
    for (int jj = 0; jj < OUT; ++jj) {
      float sj = c.q == 0 ? dzl[0][jj] + dzl[1][jj] : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sj += __shfl_xor_sync(0xffffffffu, sj, o);
      if (lane == 0 && sj != 0.f) atomicAdd(P.grads + P.b_off[L - 1] + jj, sj);
    }
    if (c.q == 0) {
      // image row: columns 0..OUT-1 = S_g * dz, rest zero
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = c.m0 + 8 * rr;
        uint32_t h0, l0, h1 = 0, l1 = 0;
        split2_f16(dzl[rr][0] * s_g, OUT > 1 ? dzl[rr][OUT > 1 ? 1 : 0] * s_g : 0.f, h0, l0);
        if (OUT == 3) split2_f16(dzl[rr][OUT - 1] * s_g, 0.f, h1, l1);
        char* g_hi = P.img.dzl + (int64_t)gt * ATOM_BYTES;
        char* g_lo = g_hi + P.img.w64_term_stride;
        const int r = m & 7;
        const int base = (m >> 3) * 1024 + r * 128;
#pragma unroll
        for (int c16 = 0; c16 < 8; ++c16) {
          const int off = base + ((c16 ^ r) << 4);
          *reinterpret_cast<uint4*>(g_hi + off) = c16 == 0 ? make_uint4(h0, h1, 0, 0) : make_uint4(0, 0, 0, 0);
          *reinterpret_cast<uint4*>(g_lo + off) = c16 == 0 ? make_uint4(l0, l1, 0, 0) : make_uint4(0, 0, 0, 0);
        }
      }
    }
    // dA_{L-1}[k] = sum_j dz[j] W_last[j][k], masked by relu'(h_{L-2}) -> dZ_{L-2}
    a_tile_reusable(c);
    if (c.tid < 64) {                                   // this tile's row-sum B operand (published by a_tile_written)
      uint4 b = make_uint4(0x3C00u, 0u, 0u, 0u);        // fp16 1.0, then zeros
      if (!ATLAS) {
        const float4 xv = *reinterpret_cast<const float4*>(P.x + ((int64_t)gt * TM + 64 * c.g + c.tid) * 4);
        __half h, lo;
        split_f16(xv.x * S_ACT, h, lo); b.y = pack2(h, lo);
        split_f16(xv.y * S_ACT, h, lo); b.z = pack2(h, lo);
        split_f16(xv.z * S_ACT, h, lo); b.w = pack2(h, lo);
      }
      *reinterpret_cast<uint4*>(rsum_b + c.g * RSUM_B_BYTES + c.tid * 16) = b;
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = 8 * i + 2 * c.q;
      const uint32_t bits0 = bits16[((int64_t)(L - 2) * P.img.rows + row0) * 16 + (col >> 4)];
      const uint32_t bits1 = bits16[((int64_t)(L - 2) * P.img.rows + row0 + 8) * 16 + (col >> 4)];
      float v[4];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int jj = 0; jj < OUT; ++jj) {
          const float w = __ldg(wlast + jj * KLAST + col + e);
          a0 = fmaf(dzl[0][jj], w, a0);
          a1 = fmaf(dzl[1][jj], w, a1);
        }
        const int sh = 15 - ((col + e) & 15);
        v[e] = ((bits0 >> sh) & 1u) ? a0 : 0.f;
        v[2 + e] = ((bits1 >> sh) & 1u) ? a1 : 0.f;
      }
      put(c.m0, col, v[0], v[1]);
      put(c.m0 + 8, col, v[2], v[3]);
    }
    a_tile_written(c);
    store_tile_rows(c, sm.a_tile, P.img.dz + (int64_t)(L - 2) * P.img.slot_stride + (int64_t)gt * TILE_IMG_BYTES,
                    P.img.term_stride);
    row_sums(L - 2);
    // ---------------- hidden layers: dA_l = dZ_l W_l  ->  dZ_{l-1}
#pragma unroll 1
    for (int l = L - 2; l >= LOW; --l) {
      uint32_t scale = 0u;
      for (int kc = 0; kc < 4; ++kc)
        consume_chunk<NST, 256>(pp, acc, a_rows + kc * ATOM_BYTES, a_rows + TILE_IMG_BYTES + kc * ATOM_BYTES, scale,
                                pending, c);
      finish_pass(pp, acc, pending, c);
      const int slot = l - 1;                           // produces dZ_{l-1}
      const bool need_img = ATLAS || slot >= 1;         // mapping dZ_0 feeds only its row sums (b0, dW0)
      a_tile_reusable(c);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = 8 * i + 2 * c.q;
        const uint32_t bits0 = bits16[((int64_t)slot * P.img.rows + row0) * 16 + (col >> 4)];
        const uint32_t bits1 = bits16[((int64_t)slot * P.img.rows + row0 + 8) * 16 + (col >> 4)];
        const int sh = 15 - (col & 15);
        float v[4];
        v[0] = ((bits0 >> sh) & 1u) ? __fmul_rn(acc[4 * i], inv_dgrad) : 0.f;
        v[1] = ((bits0 >> (sh - 1)) & 1u) ? __fmul_rn(acc[4 * i + 1], inv_dgrad) : 0.f;
        v[2] = ((bits1 >> sh) & 1u) ? __fmul_rn(acc[4 * i + 2], inv_dgrad) : 0.f;
        v[3] = ((bits1 >> (sh - 1)) & 1u) ? __fmul_rn(acc[4 * i + 3], inv_dgrad) : 0.f;
        put(c.m0, col, v[0], v[1]);
        put(c.m0 + 8, col, v[2], v[3]);
      }
      a_tile_written(c);
      if (need_img)
        store_tile_rows(c, sm.a_tile, P.img.dz + (int64_t)slot * P.img.slot_stride + (int64_t)gt * TILE_IMG_BYTES,
                        P.img.term_stride);
      row_sums(slot);
    }
    if (HAS_DPE) {
      // ---------------- dPE = dZ_0 W_0 (64 columns, 40 real) -> d(in) -> d_in += in_scale * d(in); the accumulator is
      // the first 32 registers of acc (a separate one next to it serialises the kernel's wgmma for lack of registers)
      float (&acc64)[32] = *reinterpret_cast<float(*)[32]>(&acc);
      uint32_t scale = 0u;
      for (int kc = 0; kc < 4; ++kc)
        consume_chunk<NST, 64>(pp, acc64, a_rows + kc * ATOM_BYTES, a_rows + TILE_IMG_BYTES + kc * ATOM_BYTES, scale,
                               pending, c);
      finish_pass(pp, acc64, pending, c);
      const char* pe_hi = P.img.pe + (int64_t)gt * ATOM_BYTES;
      const char* pe_lo = pe_hi + P.img.w64_term_stride;
      float din[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
      for (int i = 0; i < 5; ++i) {                      // columns < PE_COLS = 40
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * i + 2 * c.q + e;
          const int k = col >> 2, ee = col & 3;          // ee: 0,1 = sin(x0),sin(x1); 2,3 = cos(x0),cos(x1)
          const int pcol = (ee < 2) ? col + 2 : col - 2;  // d sin = cos * b,  d cos = -sin * b
          const float bk = pe_freq(k);
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const float g = __fmul_rn(acc64[4 * i + 2 * rr + e], inv_dgrad);
            const int off = atom_off(c.m0 + 8 * rr, pcol);
            const float partner = (__half2float(*reinterpret_cast<const __half*>(pe_hi + off)) +
                                   __half2float(*reinterpret_cast<const __half*>(pe_lo + off))) * (1.0f / S_ACT);
            din[rr][e] += (ee < 2) ? g * partner * bk : -g * partner * bk;     // ee & 1 == e
          }
        }
      }
      float mx = 0.f;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const float d0 = quad_sum(din[rr][0]), d1 = quad_sum(din[rr][1]);
        if (c.q == 0 && P.d_in) {
          float2* dst = reinterpret_cast<float2*>(P.d_in + (row0 + 8 * rr) * 2);
          float2 cur = P.d_in_accumulate ? *dst : make_float2(0.f, 0.f);
          cur.x += P.in_scale * d0;
          cur.y += P.in_scale * d1;
          *dst = cur;
          mx = fmaxf(mx, fmaxf(fabsf(cur.x), fabsf(cur.y)));
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      if (lane == 0 && mx > 0.f) atomicMax(P.gmax_bits + 1, __float_as_int(mx));
    }
  }
  if (c.leader) bulk_wait_all0();
  // flush the per-CTA accumulators: the two warpgroups' slices summed
  named_bar(BAR_CONSUMERS, CONSUMERS);
  static_assert(CONSUMER_WGS == 2, "the flush sums two slices");
  for (int i = threadIdx.x; i < (L - 1) * 256; i += CONSUMERS) {
    const float v = s_acc[i] + s_acc[BWD_ACC_FLOATS + i];
    if (v != 0.f) atomicAdd(P.grads + P.b_off[i >> 8] + (i & 255), v);
  }
  if (!ATLAS)
    for (int i = threadIdx.x; i < 768; i += CONSUMERS) {
      const float v = s_acc[(L - 1) * 256 + i] + s_acc[BWD_ACC_FLOATS + (L - 1) * 256 + i];
      if (v != 0.f) atomicAdd(P.grads + P.w_off[0] + i, v);
    }
}

// =============================================================================================
// weight gradients:  dW[n][k] += sum_rows dZ[row][n] * H[row][k]
// =============================================================================================
struct WgradItem {
  const char* a_img;      // M-side image, hi (lo at +a_term): 256 wide [tile][4 atoms][16 KB] or 64 wide [tile][16 KB]
  const char* b_img;      // N-side image, hi (lo at +b_term): same two shapes
  int64_t a_term, b_term;
  float* out; int ld_out; // fp32 dW block [n_rows][ld_out], columns [0, n_cols)
  int a_cols;             // 256: 128 columns per CTA of the pair, 64 per consumer warpgroup;  64: the 64x64 shape
  int b_cols;             // the MMA N: 256 or 64
  int transposed;         // 1: the M side indexes dW columns (output layer: M = last activation, N = its dZ)
  int n_rows, n_cols;     // real rows / columns of dW to write
  int cap, n_groups;      // row geometry of the network this item belongs to
  int split, n_split;     // this cluster's share of the live tiles
  int mapping;            // 1: gradients of the mapping network (second gradient scale)
  int g_fwd, g_bwd;       // row geometry: compacted flow-match groups (-1: none)
};
constexpr int MAX_WGRAD_ITEMS = 768;
struct WgradItems { WgradItem it[MAX_WGRAD_ITEMS]; int n; long long cycles[256]; };   // cycles: per-CTA duration (diagnostics)

constexpr int WG_CLUSTER = 2;            // CTAs per cluster: the pair shares (multicasts) the N-side operand
constexpr int WG_STAGE = 49152;          // 32 rows: A hi 8K | A lo 8K | B hi 16K | B lo 16K, each [atom][4 groups][1 KB]
constexpr int WG_NSTAGE = 4;
constexpr int WG_SMEM = WG_NSTAGE * WG_STAGE + 256;
constexpr int WG_THREADS = TC_THREADS;
constexpr int WG_EMPTY_ARRIVALS = WG_CLUSTER * EMPTY_ARRIVALS;   // every consumer warp of the pair frees every slot

// One work unit of this warpgroup: the M block at m0 of dW (or of dW^T), all N columns, accumulated over the unit's
// 32-row steps, then flushed with fp32 atomics.  MN-major operands: LBO = atom stride, SBO = 8-row group.
// HALF_K (the 64x64 shape): both warpgroups own the same 64 x 64 block, warpgroup g takes rows 16g..16g+15 of each step,
// so the MMA sequence has no warpgroup-dependent branch and no MMA is run twice; both flush.
template <int NB, bool HALF_K>
__device__ __forceinline__ void wgrad_unit(const WgradItem& W, int n_steps, int m0, char* stage, uint64_t* full,
                                           uint64_t* empty, uint32_t peer_empty, uint32_t& gs, const Consumer& c,
                                           float inv) {
  float acc[NB / 2];
  uint32_t scale = 0u;
  int pending = -1;
  for (int s = 0; s < n_steps; ++s, ++gs) {
    const int slot = gs % WG_NSTAGE;
    mbar_wait(&full[slot], (gs / WG_NSTAGE) & 1);
    const uint32_t sb = smem_u32(stage + slot * WG_STAGE);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < (HALF_K ? 1 : 2); ++kk) {       // 16 rows = 2 groups per MMA
      const int ks = HALF_K ? c.g : kk;
      const uint32_t a = sb + (HALF_K ? 0 : c.g * 4096) + ks * 2048;
      const uint64_t a_hi = make_desc(a, 4096, 1024), a_lo = make_desc(a + 8192, 4096, 1024);
      const uint64_t b_hi = make_desc(sb + 16384 + ks * 2048, 4096, 1024);
      const uint64_t b_lo = make_desc(sb + 32768 + ks * 2048, 4096, 1024);
      if constexpr (NB == 256) {
        wgmma_n256<1, 1>(acc, a_hi, b_hi, scale);
        wgmma_n256<1, 1>(acc, a_hi, b_lo, 1u);
        wgmma_n256<1, 1>(acc, a_lo, b_hi, 1u);
      } else {
        wgmma_n64<1, 1>(acc, a_hi, b_hi, scale);
        wgmma_n64<1, 1>(acc, a_hi, b_lo, 1u);
        wgmma_n64<1, 1>(acc, a_lo, b_hi, 1u);
      }
      scale = 1u;
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (pending >= 0 && c.warp_leader) { mbar_arrive(&empty[pending]); mbar_arrive_remote(peer_empty + pending * 8); }
    pending = slot;
  }
  wgmma_wait<0>();
  acc_fence(acc);
  if (pending >= 0 && c.warp_leader) { mbar_arrive(&empty[pending]); mbar_arrive_remote(peer_empty + pending * 8); }
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int m = m0 + 16 * c.w4 + (c.lane >> 2) + 8 * rr;
    if (!W.transposed) {                                  // dW row m, columns 8i + 2q + {0, 1}
      if (m >= W.n_rows) continue;
      float* orow = W.out + (int64_t)m * W.ld_out;
#pragma unroll
      for (int i = 0; i < NB / 8; ++i) {
        const int k = 8 * i + 2 * c.q;
        const float v0 = acc[4 * i + 2 * rr] * inv, v1 = acc[4 * i + 2 * rr + 1] * inv;
        if (((W.ld_out & 1) == 0) && k + 1 < W.n_cols) {
          atomicAdd(reinterpret_cast<float2*>(orow + k), make_float2(v0, v1));
        } else {
          if (k < W.n_cols) atomicAdd(orow + k, v0);
          if (k + 1 < W.n_cols) atomicAdd(orow + k + 1, v1);
        }
      }
    } else {                                              // dW column m, rows 8i + 2q + {0, 1}
      if (m >= W.n_cols) continue;
#pragma unroll
      for (int i = 0; i < NB / 8; ++i) {
        const int n = 8 * i + 2 * c.q;
        if (n < W.n_rows) atomicAdd(W.out + (int64_t)n * W.ld_out + m, acc[4 * i + 2 * rr] * inv);
        if (n + 1 < W.n_rows) atomicAdd(W.out + (int64_t)(n + 1) * W.ld_out + m, acc[4 * i + 2 * rr + 1] * inv);
      }
    }
  }
}

// The unit's share [t_begin, t_end) of the live tiles.  32-bit: tiles < 2^21 and n_split <= MAX_WGRAD_ITEMS.
__device__ __forceinline__ void unit_tiles(const WgradItem& W, const TileIter& ti, int& t_begin, int& t_end) {
  t_begin = ti.total * W.split / W.n_split;
  t_end = ti.total * (W.split + 1) / W.n_split;
}

// Work units ("items" = one dW GEMM restricted to a share of the rows) are dealt round-robin to clusters of two CTAs:
// cluster b processes items b, b + clusters, ... (WG_UNITS_PER_CLUSTER of them; the host builds the list).  Both CTAs
// of a cluster run the same rows and each reads its half of the M-side operand; the N-side operand is read once per
// cluster, each CTA multicasting half of it into both CTAs' rings, so every operand byte leaves HBM once.  The 64x64
// shape has no 256-wide side to split: the pair splits its row steps instead.  A ring slot is refilled only after the
// consumers of both CTAs have released it (the partner's producer writes into it), so both CTAs step through the same
// slot sequence.
__global__ void __cluster_dims__(WG_CLUSTER, 1, 1) __launch_bounds__(WG_THREADS, 1)
tc_wgrad_kernel(const WgradItems* __restrict__ items, const int* __restrict__ n_valid, const int* __restrict__ gmax_bits) {
  extern __shared__ __align__(1024) char smem_raw[];
  char* stage = smem_raw;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + WG_NSTAGE * WG_STAGE);
  uint64_t* empty = full + WG_NSTAGE;
  const int warp = warp_uniform(), lane = threadIdx.x & 31;
  const int rank = (int)cluster_ctarank(), cluster = blockIdx.x / WG_CLUSTER, n_clusters = gridDim.x / WG_CLUSTER;
  if (threadIdx.x == 0) {
    if (smem_u32(stage) & 1023u) __trap();   // the swizzled operand layouts need 1024-byte alignment
    for (int i = 0; i < WG_NSTAGE; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], WG_EMPTY_ARRIVALS); }
    fence_barrier_init();
  }
  cluster_sync();                            // the partner's barriers are initialised before any remote operation
  const int n_items = items->n;
  const long long t_start = clock64();

  if (warp >= CONSUMER_WGS * 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == CONSUMER_WGS * 4 && lane == 0) {
      uint32_t gs = 0;                                  // running stage counter across units, equal in both CTAs
      for (int it = cluster; it < n_items; it += n_clusters) {
        const WgradItem W = items->it[it];
        TileIter ti; ti.init(W.cap, W.n_groups, n_valid, W.g_fwd, W.g_bwd);
        int t_begin, t_end; unit_tiles(W, ti, t_begin, t_end);
        const int a_atoms = W.a_cols / 64, b_atoms = W.b_cols / 64;
        const bool split_rows = W.a_cols == 64;         // 64x64: CTA r takes the r-th half of the 32-row steps
        const int n_steps = (t_end - t_begin) * 4;     // a multiple of 4: the halves are equal
        const int s0 = split_rows ? rank * (n_steps / 2) : 0, s1 = split_rows ? s0 + n_steps / 2 : n_steps;
        const uint32_t tx = split_rows ? 16384 : 16384 + 2 * 4096 * b_atoms;
        for (int s = s0; s < s1; ++s, ++gs) {
          const int slot = gs % WG_NSTAGE;
          mbar_wait(&empty[slot], ((gs / WG_NSTAGE) & 1) ^ 1);
          const int gt = ti.global_tile(t_begin + (s >> 2));
          const int ch = s & 3;                        // 32-row chunk = groups 4ch .. 4ch+3 of every atom block
          char* dst = stage + slot * WG_STAGE;
          mbar_expect_tx(&full[slot], tx);
          const char* a = W.a_img + (int64_t)gt * a_atoms * ATOM_BYTES + ch * 4096;
          const char* b = W.b_img + (int64_t)gt * b_atoms * ATOM_BYTES + ch * 4096;
          if (split_rows) {
            bulk_g2s(dst, a, 4096, &full[slot]);
            bulk_g2s(dst + 8192, a + W.a_term, 4096, &full[slot]);
            bulk_g2s(dst + 16384, b, 4096, &full[slot]);
            bulk_g2s(dst + 32768, b + W.b_term, 4096, &full[slot]);
            continue;
          }
          for (int j = 0; j < 2; ++j) {                // this CTA's two atoms of A
            const int64_t off = (int64_t)(2 * rank + j) * ATOM_BYTES;
            bulk_g2s(dst + j * 4096, a + off, 4096, &full[slot]);
            bulk_g2s(dst + 8192 + j * 4096, a + W.a_term + off, 4096, &full[slot]);
          }
          if (b_atoms == 4) {                          // B: atoms 2r, 2r+1 of both terms, into both CTAs
            for (int j = 2 * rank; j < 2 * rank + 2; ++j) {
              bulk_g2s_multicast(dst + 16384 + j * 4096, b + (int64_t)j * ATOM_BYTES, 4096, &full[slot], 0x3);
              bulk_g2s_multicast(dst + 32768 + j * 4096, b + W.b_term + (int64_t)j * ATOM_BYTES, 4096, &full[slot], 0x3);
            }
          } else {                                     // B: one atom, rank 0 sends the hi term, rank 1 the lo term
            bulk_g2s_multicast(dst + 16384 + rank * 16384, b + rank * W.b_term, 4096, &full[slot], 0x3);
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<CONSUMER_REGS>();
    Consumer c; c.init();
    float s_gm, inv_gm, s_ga, inv_ga;
    grad_scales(gmax_bits, true, s_gm, inv_gm);
    grad_scales(gmax_bits, false, s_ga, inv_ga);
    const uint32_t peer_empty = mapa_shared(smem_u32(empty), rank ^ 1);
    uint32_t gs = 0;
    for (int it = cluster; it < n_items; it += n_clusters) {
      const WgradItem W = items->it[it];
      TileIter ti; ti.init(W.cap, W.n_groups, n_valid, W.g_fwd, W.g_bwd);
      int t_begin, t_end; unit_tiles(W, ti, t_begin, t_end);
      const int n_steps = (t_end - t_begin) * 4;
      if (n_steps == 0) continue;
      const float inv = (W.mapping ? inv_gm : inv_ga) * (1.0f / S_ACT);
      const int m0 = rank * 128 + c.g * 64;
      if (W.a_cols == 64) wgrad_unit<64, true>(W, n_steps / 2, 0, stage, full, empty, peer_empty, gs, c, inv);
      else if (W.b_cols == 256) wgrad_unit<256, false>(W, n_steps, m0, stage, full, empty, peer_empty, gs, c, inv);
      else wgrad_unit<64, false>(W, n_steps, m0, stage, full, empty, peer_empty, gs, c, inv);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && blockIdx.x < 256) const_cast<WgradItems*>(items)->cycles[blockIdx.x] = clock64() - t_start;
  cluster_sync();                            // no CTA exits while its partner may still arrive on its barriers
}

// =============================================================================================
// host side
// =============================================================================================
static int g_sm_count = 0;
static int sm_count() {
  if (!g_sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
    if (g_sm_count <= 0) g_sm_count = 132;
  }
  return g_sm_count;
}

static int current_device() { int d = 0; cudaGetDevice(&d); return d; }

TcNet tc_net_of(const MlpShape& s) {
  if (s.hidden != HID) return TcNet::None;
  bool skips_4_7 = true, no_skips = true;
  for (int l = 1; l < s.L; ++l) {
    skips_4_7 = skips_4_7 && s.skip[l] == (l == 4 || l == 7);
    no_skips = no_skips && !s.skip[l];
  }
  if (s.L == 6 && s.pe == 0 && s.in_dim == 3 && s.out_dim == 2 && no_skips) return TcNet::Mapping6;
  if (s.L == 4 && s.pe == 0 && s.in_dim == 3 && s.out_dim == 2 && no_skips) return TcNet::Mapping4;
  if (s.L == 8 && s.pe == 10 && s.in_dim == 2 && s.out_dim == 3 && skips_4_7) return TcNet::Atlas;
  if (s.L == 8 && s.pe == 5 && s.in_dim == 3 && s.out_dim == 1 && no_skips) return TcNet::Alpha;
  // the encoding (6 P columns) must fit the one 64-column chunk of layer 0
  const bool pe_chunk = s.pe >= 1 && s.pe <= 10;
  if (s.L == 6 && pe_chunk && s.in_dim == 3 && s.out_dim == 2 && no_skips) return TcNet::MappingPE6;
  if (s.L == 4 && pe_chunk && s.in_dim == 3 && s.out_dim == 2 && no_skips) return TcNet::MappingPE4;
  return TcNet::None;
}

// The kernel instantiations of each network, indexed by TcNet - 1.
struct NetKernels { void (*fwd)(FwdParams); void (*bwd)(BwdParams); int fwd_smem, bwd_smem; };
static const NetKernels g_kernels[] = {
    {tc_fwd_kernel<false, 6>, tc_bwd_kernel<false, 6>, KCfg<false, false>::SMEM, KCfg<false, true>::SMEM},
    {tc_fwd_kernel<false, 4>, tc_bwd_kernel<false, 4>, KCfg<false, false>::SMEM, KCfg<false, true>::SMEM},
    {tc_fwd_kernel<true, 8, 0>, tc_bwd_kernel<true, 8, 0>, KCfg<true, false>::SMEM, KCfg<true, true>::SMEM},
    {tc_fwd_kernel<true, 8, 1>, tc_bwd_kernel<true, 8, 1>, KCfg<true, false>::SMEM, KCfg<true, true>::SMEM},
    {tc_fwd_kernel<true, 6, 2>, tc_bwd_kernel<true, 6, 2>, KCfg<true, false>::SMEM, KCfg<true, true>::SMEM},
    {tc_fwd_kernel<true, 4, 2>, tc_bwd_kernel<true, 4, 2>, KCfg<true, false>::SMEM, KCfg<true, true>::SMEM},
};

// Clusters of the weight-gradient kernel that fit on each device at once (set by ensure_attrs)
static int g_wg_clusters[64];

static int ensure_attrs() {
  // cudaFuncSetAttribute is per device: remember which devices of this process have been configured
  static bool done_dev[64] = {};
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  B200_REQUIRE(dev >= 0 && dev < 64, "device ordinal %d out of range", dev);
  bool& done = done_dev[dev];
  if (done) return B200_OK;
  for (const NetKernels& k : g_kernels) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(k.fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, k.fwd_smem));
    B200_CHECK_CUDA(cudaFuncSetAttribute(k.bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, k.bwd_smem));
  }
  B200_CHECK_CUDA(cudaFuncSetAttribute(tc_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(WG_CLUSTER); cfg.blockDim = dim3(WG_THREADS); cfg.dynamicSmemBytes = WG_SMEM;
  B200_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&g_wg_clusters[dev], tc_wgrad_kernel, &cfg));
  B200_REQUIRE(g_wg_clusters[dev] > 0, "the weight-gradient kernel's %d-CTA clusters do not fit on device %d", WG_CLUSTER, dev);
  done = true;
  return B200_OK;
}

static int launch_fwd(TcNet net, const FwdParams& P, int tiles, cudaStream_t st) {
  const NetKernels& k = g_kernels[(int)net - 1];
  k.fwd<<<min(sm_count(), tiles), TC_THREADS, k.fwd_smem, st>>>(P);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

static int launch_bwd(TcNet net, const BwdParams& P, int tiles, cudaStream_t st) {
  const NetKernels& k = g_kernels[(int)net - 1];
  k.bwd<<<min(sm_count(), tiles), TC_THREADS, k.bwd_smem, st>>>(P);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// Parameter blocks as the fused step uses them; other callers override the fields that differ.
static FwdParams fill_fwd(const MlpShape& sh, const NetImages& im, const float* x, float* y, const float* params, int cap,
                          int groups, const int* n_valid) {
  FwdParams P{};
  P.x = x; P.y = y; P.params = params; P.img = im; P.cap = cap; P.n_groups = groups; P.n_valid = n_valid;
  P.in_scale = 0.5f; P.in_shift = 0.5f; P.store_images = 1; P.tanh_out = 1; P.g_fwd = P.g_bwd = -1; P.pe_freqs = sh.pe;
  for (int l = 0; l < sh.L; ++l) { P.w_off[l] = sh.w_off[l]; P.b_off[l] = sh.b_off[l]; }
  return P;
}

// The mapping of the fused step and of the render: a PE mapping encodes the raw (x, y, t) rows.
static FwdParams fill_fwd_mapping(const MlpShape& sh, const NetImages& im, const float* x, float* y, const float* params,
                                  int cap, int groups, const int* n_valid) {
  FwdParams P = fill_fwd(sh, im, x, y, params, cap, groups, n_valid);
  P.in_scale = 1.0f; P.in_shift = 0.0f;
  return P;
}

static BwdParams fill_bwd(const MlpShape& sh, const NetImages& im, const float* dy, const float* y, const float* x,
                          float* d_in, const float* params, float* grads, int cap, int groups, const int* n_valid,
                          int* gmax_bits) {
  BwdParams P{};
  P.dy = dy; P.y = y; P.x = x; P.d_in = d_in; P.params = params; P.grads = grads; P.img = im;
  P.cap = cap; P.n_groups = groups; P.n_valid = n_valid; P.gmax_bits = gmax_bits;
  P.in_scale = 0.5f; P.d_in_accumulate = 1; P.tanh_out = 1; P.g_fwd = P.g_bwd = -1;
  for (int l = 0; l < sh.L; ++l) { P.w_off[l] = sh.w_off[l]; P.b_off[l] = sh.b_off[l]; }
  return P;
}

// ---- job tables: PrepJobs for tc_prep_kernel, WgradItems for tc_wgrad_kernel
static void add_prep(PrepJobs& pj, const float* W, int ldw, int n_rows, int k0, int k_cnt, int transpose, char* dst) {
  PrepJob& j = pj.j[pj.n++];
  j.W = W; j.ldw = ldw; j.n_rows = n_rows; j.k0 = k0; j.k_cnt = k_cnt; j.transpose = transpose;
  j.hi = dst; j.lo = dst + 2 * ITEM_BYTES;
  j.f32 = nullptr; j.f32_scale = 0.f;
}
static void add_const(PrepJobs& pj, const float* src, int n, float scale, float* dst) {
  PrepJob& j = pj.j[pj.n++];
  j = PrepJob{};
  j.W = src; j.n_rows = n; j.f32 = dst; j.f32_scale = scale;
}

static void prep_jobs_for_net(PrepJobs& pj, const MlpShape& sh, const NetImages& im, const float* pp, TcNet net,
                              bool with_bwd) {
  const bool pe = tc_pe_first(net);
  const FwdConsts fc = fwd_consts(sh.L, !pe, sh.out_dim, sh.K[sh.L - 1]);
  for (int l = 0; l < sh.L - 1; ++l) add_const(pj, pp + sh.b_off[l], 256, S_ACT, im.cst + l * 256);
  if (!pe) add_const(pj, pp + sh.w_off[0], 768, S_ACT, im.cst + fc.w0);
  add_const(pj, pp + sh.w_off[sh.L - 1], sh.out_dim * sh.K[sh.L - 1], 1.0f / S_ACT, im.cst + fc.wl);
  add_const(pj, pp + sh.b_off[sh.L - 1], sh.out_dim, 1.0f, im.cst + fc.bl);
  for (int l = 0; l < sh.L; ++l) {
    char* dst = im.w_fwd + im.w_fwd_layer[l];
    if (im.n_chunks_fwd[l] == 0) continue;
    const float* W = pp + sh.w_off[l];
    int chunk = 0;
    if (l > 0) for (int kc = 0; kc < 4; ++kc) add_prep(pj, W, sh.K[l], 256, kc * 64, 64, 0, dst + (int64_t)(chunk++) * CHUNK_BYTES);
    if (pe && (l == 0 || sh.skip[l]))
      add_prep(pj, W, sh.K[l], 256, l == 0 ? 0 : 256, sh.enc, 0, dst + (int64_t)(chunk++) * CHUNK_BYTES);
  }
  if (!with_bwd) return;
  for (int l = 0; l < sh.L - 1; ++l) {
    if (l < 1 && !tc_net_has_dpe(net)) continue;
    char* dst = im.w_bwd + im.w_bwd_layer[l];
    const float* W = pp + sh.w_off[l];
    // image rows = input index k of layer l (256, or 40 for atlas layer 0), chunk over the output index n
    const int rows = (pe && l == 0) ? sh.enc : 256;
    for (int kc = 0; kc < 4; ++kc) add_prep(pj, W, sh.K[l], rows, kc * 64, 64, 1, dst + (int64_t)kc * CHUNK_BYTES);
  }
}

// wgrad work list.  Units are balanced by a per-32-row-step cost of each GEMM, indexed by the image columns of its two
// operands (a_cols + b_cols): narrow steps cost more than their bytes (barrier round trips and M = 64 MMAs do not
// shrink).  The weights are those of the one-CTA-per-SM kernel that re-read A per 64-column pass; kept, they give the same
// row shares and so the same per-unit sums.  On an H100 at a 400 W power limit the kernel takes 0.51-0.52 ms (with the
// global rigidity term) and 0.44 ms (without) at the benchmark shape, against 1.11-1.13 / 0.94 ms before; per-cluster
// busy time spreads from 0.74 to 1.11 of the mean (tools/wgrad_cluster_balance.py).
static double step_cost(int a_cols, int b_cols) {
  const int cols = a_cols + b_cols;
  return cols >= 512 ? 512.0 : (cols >= 320 ? 416.0 : 340.0);
}

struct WgProto { const char* a; int64_t a_term; int a_cols; const char* b; int64_t b_term; int b_cols; int transposed;
                 float* out; int ld; int n_rows, n_cols, groups; double bytes; int mapping; int g_fwd, g_bwd; };

static void protos_for_net(WgProto* protos, int& np, const MlpShape& sh, const NetImages& im, float* g, TcNet net,
                           int groups, int g_fwd = -1, int g_bwd = -1) {
  const bool pe = tc_pe_first(net);
  const int mapping = tc_net_is_mapping(net) ? 1 : 0;
  auto add = [&](const char* a, int64_t a_term, int a_cols, const char* b, int64_t b_term, int b_cols, float* out, int ld,
                 int n_rows, int n_cols, int transposed = 0) {
    protos[np++] = WgProto{a, a_term, a_cols, b, b_term, b_cols, transposed, out, ld, n_rows, n_cols, groups,
                           (double)groups * step_cost(a_cols, b_cols), mapping, g_fwd, g_bwd};
  };
  for (int l = 1; l <= sh.L - 2; ++l)
    add(im.dz + (int64_t)l * im.slot_stride, im.term_stride, 256, im.act + (int64_t)(l - 1) * im.slot_stride,
        im.term_stride, 256, g + sh.w_off[l], sh.K[l], 256, 256);
  // output layer: the 256-wide activation goes on the M side (split over the pair), dW is written transposed
  add(im.act + (int64_t)(sh.L - 2) * im.slot_stride, im.term_stride, 256, im.dzl, im.w64_term_stride, 64,
      g + sh.w_off[sh.L - 1], sh.K[sh.L - 1], sh.out_dim, 256, 1);
  if (pe) {
    // positional-encoding parts: layer 0 and the skip layers; output layer's skip part
    add(im.dz, im.term_stride, 256, im.pe, im.w64_term_stride, 64, g + sh.w_off[0], sh.K[0], 256, sh.enc);
    for (int l = 1; l <= sh.L - 2; ++l)
      if (sh.skip[l])
        add(im.dz + (int64_t)l * im.slot_stride, im.term_stride, 256, im.pe, im.w64_term_stride, 64, g + sh.w_off[l] + 256,
            sh.K[l], 256, sh.enc);
    if (sh.skip[sh.L - 1])
      add(im.dzl, im.w64_term_stride, 64, im.pe, im.w64_term_stride, 64, g + sh.w_off[sh.L - 1] + 256, sh.K[sh.L - 1],
          sh.out_dim, sh.enc);
  }
}

// One CTA per SM (each CTA needs most of the shared memory), in clusters of two; the GEMMs are cut into
// WG_UNITS_PER_CLUSTER x clusters units of equal cost (largest-remainder apportionment) that the clusters take
// round-robin (see tc_wgrad_kernel).  Two units per cluster keep the rows summed by one fp32 accumulator at what one
// CTA per SM summed (wgmma accumulation error grows with that length, and the ill-conditioned mapping gradients show
// it); on a 132-SM H100 the work list is the same as with one unit per SM.
constexpr int WG_UNITS_PER_CLUSTER = 2;
static int wg_clusters() { return g_wg_clusters[current_device()]; }
static void apportion_items(WgradItems& wi, const WgProto* protos, int np, int cap) {
  double total_bytes = 0;
  for (int i = 0; i < np; ++i) total_bytes += protos[i].bytes;
  const int sms = wg_clusters() * WG_UNITS_PER_CLUSTER;
  int n_split[32], used = 0;
  double frac[32];
  for (int i = 0; i < np; ++i) {
    const double want = protos[i].bytes / total_bytes * sms;
    n_split[i] = (int)want < 1 ? 1 : (int)want;
    frac[i] = want - (int)want;
    used += n_split[i];
  }
  while (used < sms) {
    int best = 0;
    for (int i = 1; i < np; ++i) if (frac[i] > frac[best]) best = i;
    ++n_split[best]; frac[best] = -1.0; ++used;
  }
  while (used > sms) {
    int best = -1;
    for (int i = 0; i < np; ++i) if (n_split[i] > 1 && (best < 0 || n_split[i] > n_split[best])) best = i;
    if (best < 0) break;
    --n_split[best]; --used;
  }
  for (int i = 0; i < np; ++i) {
    for (int sp = 0; sp < n_split[i] && wi.n < MAX_WGRAD_ITEMS; ++sp) {
      WgradItem& it = wi.it[wi.n++];
      const WgProto& pr = protos[i];
      it.a_img = pr.a; it.a_term = pr.a_term; it.a_cols = pr.a_cols;
      it.b_img = pr.b; it.b_term = pr.b_term; it.b_cols = pr.b_cols; it.transposed = pr.transposed;
      it.out = pr.out; it.ld_out = pr.ld; it.n_rows = pr.n_rows; it.n_cols = pr.n_cols;
      it.cap = cap; it.n_groups = pr.groups; it.split = sp; it.n_split = n_split[i]; it.mapping = pr.mapping;
      it.g_fwd = pr.g_fwd; it.g_bwd = pr.g_bwd;
    }
  }
}

// The tables depend only on pointers and geometry.  Callers that keep their workspace and parameter / gradient buffers
// across calls (the fused step; stand-alone calls on a persistent workspace, such as the segmentation step) take them
// from a process-wide cache: built by one eager call, kept in their own device allocations, reused inside captured
// graphs.  The render and ephemeral stand-alone calls (the IMLP class: a fresh workspace per call) upload them into
// their workspace on every call, so a recycled workspace is harmless and the cache does not grow with every call.
struct TabKey {
  int dev; const void* ws; TcNet net;   // fused step: net = Atlas (mapping + atlas) or the mapping's (pre-training)
  int pe;                               // encoding frequencies of the (mapping) network: its tables depend on them
  bool step, with_bwd; int cap, groups, g_fwd, g_bwd;
  const void* params; const void* grads;   // grads null: a stand-alone forward, served by the entry of its backward
};
struct TcTables { TabKey key; PrepJobs* d_prep = nullptr; int n_prep = -1; WgradItems* d_wg = nullptr; int n_wg = -1; };
// Captured graphs bake an entry's device pointers in, so an entry is NEVER recycled: the list only grows (each entry
// is ~75 KB of device memory; one entry per (device, workspace, row geometry, parameter buffers)).
constexpr int MAX_TABLES = 4096;
static std::vector<TcTables*> g_tabs;
static std::mutex g_tabs_mutex;
static thread_local PrepJobs g_pj;        // host side of the table being built
static thread_local WgradItems g_wi;

// The entry of `k`, or null.  `add`: a missing entry is added with no tables yet.  An entry without gradient buffer
// (made by a stand-alone forward) adopts the first one a backward brings.
static TcTables* find_tables(const TabKey& k, bool add) {
  std::lock_guard<std::mutex> lock(g_tabs_mutex);
  for (TcTables* t : g_tabs) {
    TabKey& e = t->key;
    if (e.dev == k.dev && e.ws == k.ws && e.net == k.net && e.pe == k.pe && e.step == k.step && e.with_bwd == k.with_bwd &&
        e.cap == k.cap && e.groups == k.groups && e.g_fwd == k.g_fwd && e.g_bwd == k.g_bwd && e.params == k.params &&
        (!k.grads || !e.grads || e.grads == k.grads)) {
      if (!e.grads) e.grads = k.grads;
      return t;
    }
  }
  if (!add || (int)g_tabs.size() >= MAX_TABLES) return nullptr;
  g_tabs.push_back(new TcTables{k});
  return g_tabs.back();
}

// Copies a host table to *dst: a new allocation of a cache entry (`own`) or a slot of the caller's workspace.  Either
// way it is a pageable copy made outside graph capture.  A cached table is read later from any stream, so the upload
// completes before the call returns.
template <class T> static int upload(const T& host, T** dst, bool own, cudaStream_t st) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cs);
  B200_REQUIRE(cs != cudaStreamCaptureStatusActive, "tensor-core job tables are uploaded by an eager call: run the same "
               "call once outside graph capture first (persistent workspaces only; the render is not capturable)");
  if (own) B200_CHECK_CUDA(cudaMalloc(dst, sizeof(T)));
  B200_CHECK_CUDA(cudaMemcpyAsync(*dst, &host, sizeof(T), cudaMemcpyHostToDevice, st));
  if (own) B200_CHECK_CUDA(cudaStreamSynchronize(st));
  return B200_OK;
}

// the compacted flow-match groups of the fused step's mapping batch: G_FWD = 5, G_BWD = 6 when it has them
static int step_g_fwd(const TcStep& s) { return (s.flow_groups && s.n_groups > 6) ? 5 : -1; }
static int step_g_bwd(const TcStep& s) { return (s.flow_groups && s.n_groups > 6) ? 6 : -1; }

static TabKey step_key(const TcStep& s) {
  return TabKey{current_device(), s.plan->base, s.y_atlas ? TcNet::Atlas : tc_net_of(*s.ms), s.ms->pe, true, true, s.cap,
                s.n_groups, step_g_fwd(s), step_g_bwd(s), s.params, s.grads};
}

static bool step_shapes_ok(const TcStep& s) {
  const TcNet m = tc_net_of(*s.ms);
  return (m == TcNet::Mapping6 || m == TcNet::MappingPE6) && tc_net_of(*s.as) == TcNet::Atlas;
}

// The weight images depend only on the parameters, so their preparation runs on a side stream, forked from the
// caller's stream before the sampling kernels and joined before the first fused kernel (also under capture: the
// fork / join become parallel branches of the graph).
struct SideStream { cudaStream_t stream = nullptr; cudaEvent_t fork = nullptr, join = nullptr; bool pending = false; };
static SideStream g_side[64];

int tc_begin_step(const TcStep& s, cudaStream_t st) {
  B200_PROPAGATE(ensure_attrs());
  TcTables* tab = find_tables(step_key(s), true);
  B200_REQUIRE(tab, "too many distinct tensor-core workspaces in one process (%d)", MAX_TABLES);
  if (tab->n_wg < 0) {
    B200_REQUIRE(step_shapes_ok(s), "tensor-core path is specialised to the two stage-1 networks (6-layer mapping, "
                 "with or without positional encoding, and the atlas)");
    const TcLayout lay = layout_of(s);
    const TcNet mnet = tc_net_of(*s.ms);
    const bool atlas = s.y_atlas != nullptr;
    // ---- forward / dgrad weight images (the atlas network only where it is evaluated: not in pre-training)
    g_pj.n = 0;
    prep_jobs_for_net(g_pj, *s.ms, lay.map, s.params, mnet, true);
    if (atlas) prep_jobs_for_net(g_pj, *s.as, lay.atl, s.params + s.ms->total, TcNet::Atlas, true);
    if (g_pj.n > MAX_PREP_JOBS) { set_error("table overflow"); return B200_ERR_INVALID; }
    // ---- wgrad items
    WgProto protos[32]; int np = 0;
    protos_for_net(protos, np, *s.ms, lay.map, s.grads, mnet, s.n_groups, step_g_fwd(s), step_g_bwd(s));
    if (atlas) protos_for_net(protos, np, *s.as, lay.atl, s.grads + s.ms->total, TcNet::Atlas, 3);
    g_wi.n = 0;
    apportion_items(g_wi, protos, np, s.cap);
    B200_PROPAGATE(upload(g_pj, &tab->d_prep, true, st));
    B200_PROPAGATE(upload(g_wi, &tab->d_wg, true, st));
    tab->n_prep = g_pj.n; tab->n_wg = g_wi.n;
  }
  SideStream& sd = g_side[current_device()];
  if (!sd.stream) {
    B200_CHECK_CUDA(cudaStreamCreateWithFlags(&sd.stream, cudaStreamNonBlocking));
    B200_CHECK_CUDA(cudaEventCreateWithFlags(&sd.fork, cudaEventDisableTiming));
    B200_CHECK_CUDA(cudaEventCreateWithFlags(&sd.join, cudaEventDisableTiming));
  }
  B200_CHECK_CUDA(cudaEventRecord(sd.fork, st));
  B200_CHECK_CUDA(cudaStreamWaitEvent(sd.stream, sd.fork, 0));
  // weight images of both networks — every step, since Adam changed the parameters
  tc_prep_kernel<<<tab->n_prep * 4, 128, 0, sd.stream>>>(tab->d_prep);
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(cudaEventRecord(sd.join, sd.stream));
  sd.pending = true;
  return B200_OK;
}

int tc_step_forward(const TcStep& s, cudaStream_t st) {
  const TcLayout lay = layout_of(s);
  SideStream& sd = g_side[current_device()];
  if (!sd.pending) B200_PROPAGATE(tc_begin_step(s, st));     // callers that did not fork earlier
  B200_CHECK_CUDA(cudaStreamWaitEvent(st, sd.join, 0));
  sd.pending = false;
  FwdParams pm = fill_fwd_mapping(*s.ms, lay.map, s.x_map, s.uv, s.params, s.cap, s.n_groups, s.counters);
  pm.g_fwd = step_g_fwd(s); pm.g_bwd = step_g_bwd(s);
  timer_begin(TAG_MAP_FWD, st);
  B200_PROPAGATE(launch_fwd(tc_net_of(*s.ms), pm, s.n_groups * (s.cap / TM), st));
  timer_end(TAG_MAP_FWD, st);
  if (s.y_atlas) {
    const FwdParams pa = fill_fwd(*s.as, lay.atl, s.uv, s.y_atlas, s.params + s.ms->total, s.cap, 3, s.counters);
    timer_begin(TAG_ATLAS_FWD, st);
    B200_PROPAGATE(launch_fwd(TcNet::Atlas, pa, 3 * (s.cap / TM), st));
    timer_end(TAG_ATLAS_FWD, st);
  }
  return B200_OK;
}

static const WgradItems* g_last_wg = nullptr;
static int g_last_wg_n = 0;

// diagnostics: per-CTA cycle counts and the dW shape (rows, columns of its image operands) and n_split of the first item
// each CTA ran in the last weight-gradient launch; CTAs 2c and 2c + 1 form cluster c
int tc_debug_wgrad(long long* cycles, int* shapes, int max_ctas) {
  if (!g_last_wg) { set_error("no weight-gradient launch yet"); return -1; }
  static WgradItems host;
  if (cudaMemcpy(&host, g_last_wg, sizeof(WgradItems), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  const int n = g_last_wg_n < max_ctas ? g_last_wg_n : max_ctas;
  for (int i = 0; i < n; ++i) {
    const WgradItem& it = host.it[i / WG_CLUSTER];
    cycles[i] = host.cycles[i];
    shapes[3 * i] = it.transposed ? it.b_cols : it.a_cols; shapes[3 * i + 1] = it.transposed ? it.a_cols : it.b_cols;
    shapes[3 * i + 2] = it.n_split;
  }
  return n;
}

// An entry is correct whenever its key matches (the key names every pointer and extent its tables hold), but it
// outlives the buffers it names.  A process that fits one trainer after another (one atlas per clip of a long video)
// would keep every earlier trainer's entries: device memory outside the caller's allocator, and a slot each towards
// MAX_TABLES.  The owner of a parameter buffer frees its entries here once no graph that bakes them in is replayed.
int tc_release_tables(const void* begin, const void* end) {
  std::lock_guard<std::mutex> lock(g_tabs_mutex);
  const int dev = current_device();
  int n = 0;
  for (size_t i = 0; i < g_tabs.size();) {
    TcTables* t = g_tabs[i];
    const void* p = t->key.params;
    if (t->key.dev != dev || p < begin || p >= end) { ++i; continue; }
    if (t->d_wg && t->d_wg == g_last_wg) { g_last_wg = nullptr; g_last_wg_n = 0; }
    B200_CHECK_CUDA(cudaFree(t->d_prep));
    B200_CHECK_CUDA(cudaFree(t->d_wg));
    delete t;
    g_tabs.erase(g_tabs.begin() + i);
    ++n;
  }
  return n;
}

int tc_cached_tables() {
  std::lock_guard<std::mutex> lock(g_tabs_mutex);
  return (int)g_tabs.size();
}

// grid of a weight-gradient launch: as many clusters as fit on the device at once, at most one per work unit
static int wgrad_grid(int n_items) { return WG_CLUSTER * min(n_items, wg_clusters()); }

int tc_step_backward(const TcStep& s, cudaStream_t st) {
  const TcLayout lay = layout_of(s);
  const TcTables* tab = find_tables(step_key(s), false);
  B200_REQUIRE(tab && tab->n_wg >= 0, "tensor-core backward called before forward");
  int* gmax = const_cast<int*>(s.counters) + 3;
  if (s.y_atlas) {
    const BwdParams pa = fill_bwd(*s.as, lay.atl, s.d_y, s.y_atlas, nullptr, const_cast<float*>(s.d_uv),
                                  s.params + s.ms->total, s.grads + s.ms->total, s.cap, 3, s.counters, gmax);
    timer_begin(TAG_ATLAS_BWD, st);
    B200_PROPAGATE(launch_bwd(TcNet::Atlas, pa, 3 * (s.cap / TM), st));
    timer_end(TAG_ATLAS_BWD, st);
  }
  BwdParams pm = fill_bwd(*s.ms, lay.map, s.d_uv, s.uv, s.x_map, nullptr, s.params, s.grads, s.cap, s.n_groups,
                          s.counters, gmax);
  pm.g_fwd = step_g_fwd(s); pm.g_bwd = step_g_bwd(s);
  timer_begin(TAG_MAP_BWD, st);
  B200_PROPAGATE(launch_bwd(tc_net_of(*s.ms), pm, s.n_groups * (s.cap / TM), st));
  timer_end(TAG_MAP_BWD, st);
  timer_begin(TAG_WGRAD, st);
  g_last_wg = tab->d_wg; g_last_wg_n = wgrad_grid(tab->n_wg);
  tc_wgrad_kernel<<<wgrad_grid(tab->n_wg), WG_THREADS, WG_SMEM, st>>>(tab->d_wg, s.counters, gmax);
  timer_end(TAG_WGRAD, st);
  B200_CHECK_LAUNCH();
  return B200_OK;
}


// ---------------------------------------------------------------------------------------------
// inference: mapping -> atlas on `rows` coordinate rows, no activation images (full-video render,
// evaluate.py:640-708).  Workspace: [PrepJobs table][forward weight images of both networks].
// ---------------------------------------------------------------------------------------------

static int64_t plan_infer(const MlpShape& ms, const MlpShape& as, char* base, NetImages* im_map, NetImages* im_atl,
                          PrepJobs** d_prep) {
  char* p = align_tc(base);
  *d_prep = reinterpret_cast<PrepJobs*>(carve_tc(p, sizeof(PrepJobs)));
  *im_map = NetImages{}; *im_atl = NetImages{};
  plan_fwd_weights(ms, tc_net_of(ms), p, im_map);
  plan_fwd_weights(as, TcNet::Atlas, p, im_atl);
  return p - base;
}

int64_t tc_infer_workspace_bytes(const MlpShape& ms, const MlpShape& as) {
  NetImages a, b; PrepJobs* d;
  return plan_infer(ms, as, nullptr, &a, &b, &d) + 2048;
}

int tc_infer_forward(const MlpShape& ms, const MlpShape& as, const float* params, const float* x_map, float* uv,
                     float* y, int64_t rows, char* ws, cudaStream_t st) {
  B200_PROPAGATE(ensure_attrs());
  const TcNet mnet = tc_net_of(ms);
  B200_REQUIRE((mnet == TcNet::Mapping6 || mnet == TcNet::MappingPE6) && tc_net_of(as) == TcNet::Atlas,
               "tensor-core path is specialised to the two stage-1 networks");
  B200_REQUIRE(rows > 0 && rows % TM == 0 && rows / TM < (1 << 24), "rows must be a positive multiple of %d", TM);
  NetImages im_map, im_atl; PrepJobs* d_prep;
  plan_infer(ms, as, ws, &im_map, &im_atl, &d_prep);
  // one prep launch for both networks; the job table is rebuilt in the workspace on every call (4 KB)
  g_pj.n = 0;
  prep_jobs_for_net(g_pj, ms, im_map, params, mnet, false);
  prep_jobs_for_net(g_pj, as, im_atl, params + ms.total, TcNet::Atlas, false);
  B200_PROPAGATE(upload(g_pj, &d_prep, false, st));
  tc_prep_kernel<<<g_pj.n * 4, 128, 0, st>>>(d_prep);
  B200_CHECK_LAUNCH();
  const int tiles = (int)(rows / TM);
  FwdParams pm = fill_fwd_mapping(ms, im_map, x_map, uv, params, (int)rows, 1, nullptr);
  pm.store_images = 0;
  B200_PROPAGATE(launch_fwd(mnet, pm, tiles, st));
  FwdParams pa = fill_fwd(as, im_atl, uv, y, params + ms.total, (int)rows, 1, nullptr);
  pa.store_images = 0;
  return launch_fwd(TcNet::Atlas, pa, tiles, st);
}

// ---------------------------------------------------------------------------------------------
// stand-alone evaluation of ONE of the networks with autograd support: what the `IMLP` class needs
// (implicit_neural_networks.py:62-81 forward + the autograd of its Linear/ReLU/tanh/skip stack).
// Workspace: [PrepJobs][WgradItems][images of the network]; the two table slots serve ephemeral callers.
// ---------------------------------------------------------------------------------------------
struct SinglePlan { PrepJobs* d_prep; WgradItems* d_wg; NetImages im; int64_t bytes; };

static void plan_single(const MlpShape& sh, TcNet net, int64_t rows, char* base, SinglePlan* out) {
  char* p = align_tc(base);
  out->d_prep = reinterpret_cast<PrepJobs*>(carve_tc(p, sizeof(PrepJobs)));
  out->d_wg = reinterpret_cast<WgradItems*>(carve_tc(p, sizeof(WgradItems)));
  plan_net(sh, rows, net, p, &out->im);
  out->bytes = p - base;
}

int64_t tc_single_workspace_bytes(const MlpShape& sh, TcNet net, int64_t rows) {
  SinglePlan pl{};
  plan_single(sh, net, rows, nullptr, &pl);
  return pl.bytes + 2048;
}

// ---------------------------------------------------------------------------------------------
// diagnostics: where the images of one network lie, from the plans the kernels' launches use
// ---------------------------------------------------------------------------------------------
static void image_offsets(const NetImages& im, const char* ws, int64_t* out) {
  auto at = [&](const void* p) { return p ? (int64_t)(reinterpret_cast<const char*>(p) - ws) : (int64_t)-1; };
  out[0] = at(im.w_fwd); out[1] = at(im.w_bwd); out[2] = at(im.cst); out[3] = at(im.act);
  out[4] = at(im.dz); out[5] = at(im.pe); out[6] = at(im.dzl); out[7] = at(im.bits);
  out[8] = im.slot_stride; out[9] = im.term_stride; out[10] = im.w64_term_stride; out[11] = im.rows;
  for (int l = 0; l < B200_MAX_LAYERS; ++l) {
    out[12 + l] = im.w_fwd_layer[l];
    out[12 + B200_MAX_LAYERS + l] = im.n_chunks_fwd[l];
    out[12 + 2 * B200_MAX_LAYERS + l] = im.w_bwd_layer[l];
  }
}

void tc_single_image_offsets(const MlpShape& sh, TcNet net, int64_t rows, char* tc_ws, const char* ws, int64_t* out) {
  SinglePlan pl{};
  plan_single(sh, net, rows, tc_ws, &pl);
  image_offsets(pl.im, ws, out);
}

void tc_step_image_offsets(const MlpShape& ms, const MlpShape& as, const TcPlan& plan, bool atlas, const char* ws,
                           int64_t* out) {
  TcStep s{};
  s.ms = &ms; s.as = &as; s.plan = &plan;
  const TcLayout lay = layout_of(s);
  image_offsets(atlas ? lay.atl : lay.map, ws, out);
}

static int check_single(const MlpShape& sh, TcNet net, const TcRows& r) {
  B200_PROPAGATE(ensure_attrs());
  B200_REQUIRE(net != TcNet::None && tc_net_of(sh) == net, "tensor-core IMLP: the shape is not the network it is "
               "called for (mapping 3-256x{4,2}-2, atlas 2-PE10-256x6-3 with skips 4, 7, alpha 3-PE5-256x6-1, "
               "PE mapping 3-PE{1..10}-256x{4,2}-2)");
  B200_REQUIRE(r.cap > 0 && r.cap % TM == 0 && r.groups > 0 && r.rows() / TM < (1 << 20),
               "rows must be a positive multiple of %d", TM);
  B200_REQUIRE(r.g_fwd < 0 || r.g_bwd < 0 || r.g_fwd != r.g_bwd, "the two compacted groups must differ");
  return B200_OK;
}

// The tables of a stand-alone call: the cache entry of a persistent workspace, else the workspace's own slots.  The
// weight-gradient items depend on the row geometry (cap, groups, compacted groups), not on the counts themselves.
static TcTables* single_tables(TcTables& eph, const MlpShape& sh, TcNet net, const char* ws, const TcRows& r,
                               const float* params, const float* grads, bool training, bool persistent) {
  if (!persistent) return &eph;
  return find_tables(TabKey{current_device(), ws, net, sh.pe, false, training, r.cap, r.groups, r.g_fwd, r.g_bwd,
                            params, grads}, true);
}

static FwdParams fill_single_fwd(const MlpShape& sh, const NetImages& im, const float* x, float* y, const float* params,
                                 const TcRows& r) {
  FwdParams P = fill_fwd(sh, im, x, y, params, r.cap, r.groups, r.counters);
  P.g_fwd = r.g_fwd; P.g_bwd = r.g_bwd;
  return P;
}

// x: mapping [rows][4], atlas [rows][2] (network input itself).  y: [rows][out_dim].  Only the tiles holding live rows
// of `r` are evaluated; the other rows of y are left as they were.
int tc_single_forward(const MlpShape& sh, TcNet net, const float* params, const float* x, float* y, const TcRows& r,
                      bool training, char* ws, bool persistent, cudaStream_t st) {
  B200_PROPAGATE(check_single(sh, net, r));
  const int64_t rows = r.rows();
  SinglePlan pl{};
  plan_single(sh, net, rows, ws, &pl);
  TcTables eph{}; eph.d_prep = pl.d_prep;
  TcTables* tab = single_tables(eph, sh, net, ws, r, params, nullptr, training, persistent);
  B200_REQUIRE(tab, "too many distinct tensor-core workspaces in one process (%d)", MAX_TABLES);
  if (tab->n_prep < 0) {
    g_pj.n = 0;
    prep_jobs_for_net(g_pj, sh, pl.im, params, net, training);
    B200_PROPAGATE(upload(g_pj, &tab->d_prep, persistent, st));
    tab->n_prep = g_pj.n;
  }
  tc_prep_kernel<<<tab->n_prep * 4, 128, 0, st>>>(tab->d_prep);
  B200_CHECK_LAUNCH();
  FwdParams P = fill_single_fwd(sh, pl.im, x, y, params, r);
  P.in_scale = 1.0f; P.in_shift = 0.0f; P.store_images = training ? 1 : 0; P.tanh_out = sh.tanh_out ? 1 : 0;
  return launch_fwd(net, P, (int)(rows / TM), st);
}

// after tc_single_forward(training) on the same workspace and row geometry.  y: the saved outputs, dy [rows][out_dim]
// (zero in the padding rows of the live tiles), gmax: device int holding the bits of max|dy| (>= 0), d_in: atlas only,
// [rows][2] or null (written for the live tiles only).
int tc_single_backward(const MlpShape& sh, TcNet net, const float* params, float* grads, const float* x,
                       const float* y, const float* dy, float* d_in, int* gmax2, const TcRows& r, char* ws,
                       bool persistent, cudaStream_t st) {
  B200_PROPAGATE(check_single(sh, net, r));
  const int64_t rows = r.rows();
  SinglePlan pl{};
  plan_single(sh, net, rows, ws, &pl);
  TcTables eph{}; eph.d_wg = pl.d_wg;
  TcTables* tab = single_tables(eph, sh, net, ws, r, params, grads, true, persistent);
  B200_REQUIRE(tab, "too many distinct tensor-core workspaces in one process (%d)", MAX_TABLES);
  if (tab->n_wg < 0) {
    WgProto protos[32]; int np = 0;
    protos_for_net(protos, np, sh, pl.im, grads, net, r.groups, r.g_fwd, r.g_bwd);
    g_wi.n = 0;
    apportion_items(g_wi, protos, np, r.cap);
    B200_PROPAGATE(upload(g_wi, &tab->d_wg, persistent, st));
    tab->n_wg = g_wi.n;
  }
  // gmax2: [0] atlas scale, [1] mapping scale
  BwdParams P = fill_bwd(sh, pl.im, dy, y, x, d_in, params, grads, r.cap, r.groups, r.counters, gmax2);
  P.in_scale = 1.0f; P.d_in_accumulate = 0; P.tanh_out = sh.tanh_out ? 1 : 0; P.g_fwd = r.g_fwd; P.g_bwd = r.g_bwd;
  B200_PROPAGATE(launch_bwd(net, P, (int)(rows / TM), st));
  tc_wgrad_kernel<<<wgrad_grid(tab->n_wg), WG_THREADS, WG_SMEM, st>>>(tab->d_wg, r.counters, gmax2);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // namespace b200
