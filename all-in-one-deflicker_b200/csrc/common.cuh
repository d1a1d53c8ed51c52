// Shared declarations of libb200deflicker: error plumbing, MLP layout, internal launchers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200_deflicker.h"

namespace b200 {

void set_error(const char* fmt, ...);
void count_launch();

// Optional device timer around ONE tagged launch site (b200_set_kernel_timer): bench.py uses it to
// time the dominant kernel inside the replayed step.  Works under stream capture (external events).
enum KernelTag { TAG_NONE = 0, TAG_MAP_FWD = 1, TAG_MAP_BWD = 2, TAG_ATLAS_FWD = 3, TAG_ATLAS_BWD = 4,
                 TAG_WGRAD = 5, TAG_ADAM = 6 };
void timer_begin(int tag, cudaStream_t st);
void timer_end(int tag, cudaStream_t st);

#define B200_CHECK_CUDA(expr)                                                          \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      b200::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return B200_ERR_CUDA;                                                            \
    }                                                                                  \
  } while (0)

#define B200_CHECK_LAUNCH()                                                            \
  do {                                                                                 \
    b200::count_launch();                                                              \
    cudaError_t _e = cudaPeekAtLastError();                                            \
    if (_e != cudaSuccess) {                                                           \
      b200::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return B200_ERR_CUDA;                                                            \
    }                                                                                  \
  } while (0)

#define B200_REQUIRE(cond, ...)                                                        \
  do {                                                                                 \
    if (!(cond)) {                                                                     \
      b200::set_error(__VA_ARGS__);                                                    \
      return B200_ERR_INVALID;                                                         \
    }                                                                                  \
  } while (0)

#define B200_PROPAGATE(expr)                                                           \
  do {                                                                                 \
    int _rc = (expr);                                                                  \
    if (_rc != B200_OK) return _rc;                                                    \
  } while (0)

constexpr int kTileRows = 128;  // row granularity of every batched buffer (MMA M)

inline int64_t round_up(int64_t v, int64_t m) { return (v + m - 1) / m * m; }

// Resolved shape of one IMLP.
struct MlpShape {
  int L = 0;                        // layers
  int in_dim = 0, out_dim = 0, hidden = 0, pe = 0, enc = 0;
  bool tanh_out = true;
  int K[B200_MAX_LAYERS];           // fan-in of layer i (including the skip part)
  int N[B200_MAX_LAYERS];           // fan-out
  bool skip[B200_MAX_LAYERS];
  int64_t w_off[B200_MAX_LAYERS], b_off[B200_MAX_LAYERS];
  int64_t total = 0;                // padded float count
};

int resolve_mlp(const B200MlpDesc* d, MlpShape* s);   // 0 or B200_ERR_INVALID
const B200MlpDesc& mapping_desc();
const B200MlpDesc& atlas_desc();

// Validity of the rows of a group-major batch: group g holds rows [g*cap, g*cap + *n_valid).
// n_valid == nullptr means every row is valid.
struct RowSpan {
  int64_t rows = 0;        // total rows (= groups * cap)
  int64_t cap = 0;         // rows per group (multiple of kTileRows) — 0: single group of `rows`
  const int* n_valid = nullptr;
};

// Scratch carved out of the caller's workspace for one network evaluation.
struct MlpScratch {
  float* act[B200_MAX_LAYERS];      // input of layer i: [rows, K[i]]  (post-ReLU, skip part appended)
  float* y = nullptr;               // network output after tanh [rows, out_dim]
  float* dz[2] = {nullptr, nullptr};// ping-pong gradient buffers [rows, max(hidden, enc, out_dim)]
  int64_t bytes = 0;
};
int64_t plan_mlp_scratch(const MlpShape& s, int64_t rows, bool training, char* base, MlpScratch* out);

// ---- SIMT fp32 path (mlp_simt.cu)
int simt_mlp_forward(const MlpShape& s, const float* params, const float* x, int ldx, const RowSpan& span,
                     const MlpScratch& sc, float* y, cudaStream_t st);
// dy: gradient w.r.t. the network output [rows, out_dim]; dx (optional): gradient w.r.t. the
// encoded input act[0] ([rows, enc] when pe > 0, else [rows, in_dim] with leading dim ldx_out)
int simt_mlp_backward(const MlpShape& s, const float* params, const float* x, int ldx, const RowSpan& span,
                      const MlpScratch& sc, const float* dy, float* dparams, float* d_in, int ld_din,
                      cudaStream_t st);

// ---- elementwise helpers (atlas_kernels.cu)
int launch_pe_forward(const float* uv, int ld_uv, float scale, float shift, int in_dim, int freqs,
                      float* out0, int ld0, float* const* skip_outs, const int* skip_lds, int n_skip,
                      int skip_col, const RowSpan& span, cudaStream_t st);
int launch_pe_backward(const float* pe, int ld_pe, const float* dpe, int ld_dpe, int in_dim, int freqs,
                       float scale, float* d_uv, int ld_duv, int accumulate, const RowSpan& span,
                       cudaStream_t st);

}  // namespace b200
