// Internal launchers of the atlas-loop kernels (atlas_kernels.cu), used by c_api.cu.
#pragma once
#include "common.cuh"

namespace b200 {

struct LossConfig;

constexpr int TARGET_FLOATS = 12;   // per sample: rgb(3) dx(3) dy(3) wf wb pad

struct SampleGeom {
  float half_larger;   // fp32(max(resx,resy) / 2)   src/stage1_neural_atlas.py:136,169
  float half_resx;     // fp32(resx / 2)             loss_utils.py:138 (gradient-loss rows)
  float half_frames;   // fp32(number_of_frames / 2)
  float d_local;       // derivative_amount
  float d_global;      // global_rigidity_derivative_amount_fg
};

int launch_video_pack(const float* fr, const float* dx, const float* dy, const float* ff, const float* fb,
                      const float* mf, const float* mb, int H, int W, int T, int t_begin, int t_end,
                      float* rec, uint32_t* bits_f, uint32_t* bits_b, cudaStream_t st);
// matte: bootstrapping matte of the resident frames, frame-major [t_end - t_begin][H][W] (segmentation variant), copied
// into target column 11; null: column 11 stays zero (single-layer variant)
int launch_select_sample(const int64_t* indices, int B, const B200Video& vid, const SampleGeom& geo, int cap,
                         int n_groups, int* counters, int* list, float* x_map, float* targets,
                         cudaStream_t st, const float* matte = nullptr);
int launch_pretrain_sample(const int64_t* ys, const int64_t* xs, int B, int cap, float half_larger,
                           float t_norm, float* x_map, int* counters, cudaStream_t st);
int launch_pretrain_loss(const float* x_map, const float* uv, int B, int cap, float uv_scale, float* d_uv,
                         float* losses, int* counters, cudaStream_t st);
int launch_loss(const float* uv, const float* y_atlas, const float* targets, int* counters, int cap,
                int n_groups, const LossConfig& cfg, float* d_uv, float* d_y, float* losses,
                cudaStream_t st);
int launch_adam(float* p, const float* g, float* m, float* v, int64_t n, double lr, double b1, double b2,
                double eps, float grad_scale, int64_t* step, cudaStream_t st);
int launch_dp_adam(const B200DpComm& comm, float* m, float* v, int64_t n_params, int64_t n_total, double lr,
                   double b1, double b2, double eps, int64_t* step, unsigned long long* epoch, cudaStream_t st);
int launch_pack_rows(const float* src, int ld_src, int cols, float* dst, int ld_dst, int64_t rows, int64_t rows_pad,
                     cudaStream_t st);
int launch_absmax(const float* src, int64_t n, int* out_bits, cudaStream_t st);
int launch_render_rows(int W, float half_larger, float t_norm, int64_t pix_begin, int64_t count,
                       int64_t rows_padded, float* x_map, cudaStream_t st);
int launch_render_out(const float* y, int64_t count, float* rgb, uint8_t* u8, cudaStream_t st);

}  // namespace b200
