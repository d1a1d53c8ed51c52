// Interface between c_api.cu and the tensor-core (wgmma) path (mlp_tc.cu).
#pragma once
#include "common.cuh"

namespace b200 {

// The networks the tensor-core kernels are instantiated for: the stage-1 mapping (3-256x4-2), the background mapping of
// the segmentation variant (3-256x2-2), the atlas (2-PE10-256x6-3, skips 4, 7), the alpha network of the
// segmentation variant (3-PE5-256x6-1) and the position-encoded mappings (3-PE P-256x{4,2}-2, P = 1..10:
// use_positional_encoding_mapping1/2 of the scripts' configs).
enum class TcNet { None, Mapping6, Mapping4, Atlas, Alpha, MappingPE6, MappingPE4 };
TcNet tc_net_of(const MlpShape& s);
// atlas, alpha and the PE mappings: the positional encoding feeds layer 0, which runs on the tensor cores
inline bool tc_pe_first(TcNet n) {
  return n == TcNet::Atlas || n == TcNet::Alpha || n == TcNet::MappingPE6 || n == TcNet::MappingPE4;
}
// the atlas back-propagates to its input (uv) through the encoding; the other networks' inputs are pixel coordinates
inline bool tc_net_has_dpe(TcNet n) { return n == TcNet::Atlas; }
// the 3 -> 2 mappings: their gradients take the second gradient scale (max |dL/duv|)
inline bool tc_net_is_mapping(TcNet n) {
  return n == TcNet::Mapping6 || n == TcNet::Mapping4 || n == TcNet::MappingPE6 || n == TcNet::MappingPE4;
}

// Buffers of the tensor-core path, carved from the caller's workspace (see mlp_tc.cu).
struct TcPlan {
  char* base = nullptr;
  int64_t bytes = 0;
  int64_t rows_map = 0, rows_atlas = 0;
};

// The fused step and the render take the 6-layer mapping, with or without positional encoding (tc_net_of(ms) is
// Mapping6 or MappingPE6), and the atlas.
struct TcStep {
  const MlpShape* ms; const MlpShape* as;
  const TcPlan* plan;
  const float* params; float* grads;
  const float* x_map;        // [n_groups*cap][4]
  float* uv;                 // [n_groups*cap][2]  mapping output
  float* y_atlas;            // [3*cap][3]         atlas output; null: pre-training (mapping only)
  const float* d_uv;         // [n_groups*cap][2]  direct gradient of the loss head
  const float* d_y;          // [3*cap][3]
  int cap, n_groups;
  const int* counters;
  int flow_groups;           // 1: groups 5 / 6 of the mapping batch hold counters[5] / counters[6] compacted rows
};

int64_t tc_plan(const MlpShape& ms, const MlpShape& as, int64_t rows_map, int64_t rows_atlas, char* base,
                TcPlan* out);
int tc_begin_step(const TcStep& s, cudaStream_t st);      // optional: start the weight-image preparation early (side stream)
int tc_step_forward(const TcStep& s, cudaStream_t st);    // mapping on all groups, atlas on groups 0..2
int tc_step_backward(const TcStep& s, cudaStream_t st);   // all parameter gradients

// inference (render): x_map [rows][4] -> uv [rows][2] -> y [rows][3]; rows a multiple of 128; ws >= tc_infer_workspace_bytes
int64_t tc_infer_workspace_bytes(const MlpShape& ms, const MlpShape& as);
int tc_infer_forward(const MlpShape& ms, const MlpShape& as, const float* params, const float* x_map, float* uv,
                     float* y, int64_t rows, char* ws, cudaStream_t st);

// Rows of a stand-alone call: `groups` groups of `cap` rows each, group-major.  counters null: every row is live.
// Otherwise (device counters of the sampling kernels) the first counters[0] rows of each group are live, except in
// the compacted groups g_fwd / g_bwd (-1: none), whose first counters[5] / counters[6] rows are; the kernels visit only
// the 128-row tiles that hold live rows.
struct TcRows {
  int cap = 0, groups = 1;
  const int* counters = nullptr;
  int g_fwd = -1, g_bwd = -1;
  int64_t rows() const { return (int64_t)cap * groups; }
};
inline TcRows tc_all_rows(int64_t rows) { TcRows r; r.cap = (int)rows; return r; }

// stand-alone IMLP (one network, autograd): see mlp_tc.cu
int64_t tc_single_workspace_bytes(const MlpShape& sh, TcNet net, int64_t rows);
// persistent: the caller keeps this workspace and these parameter / gradient buffers across calls -> job tables are
// cached in their own device allocations and the calls become graph-capturable after one eager call
int tc_single_forward(const MlpShape& sh, TcNet net, const float* params, const float* x, float* y, const TcRows& r,
                      bool training, char* ws, bool persistent, cudaStream_t st);
int tc_single_backward(const MlpShape& sh, TcNet net, const float* params, float* grads, const float* x,
                       const float* y, const float* dy, float* d_in, int* gmax2, const TcRows& r, char* ws,
                       bool persistent, cudaStream_t st);

// b200_mlp_forward / b200_mlp_backward on a group-major batch whose live rows `live` describes (live.rows() rows):
// on the tensor cores only the tiles holding live rows are evaluated (the fp32 path evaluates every row).  The rows
// of dy outside the live ones must be zero or lie in tiles without live rows.  Used by the segmentation step.
int mlp_forward_rows(const B200MlpDesc* d, const float* params, const float* x, float* y, const TcRows& live,
                     int training, int precision, void* ws, int64_t ws_bytes, cudaStream_t st);
int mlp_backward_rows(const B200MlpDesc* d, const float* params, const float* x, const float* dy, float* dparams,
                      float* dx, const TcRows& live, int precision, void* ws, int64_t ws_bytes, cudaStream_t st);

// Scope guard used by entry points that own a persistent workspace (the segmentation step): while alive,
// b200_mlp_forward / backward calls made by this thread use the cached-table path above.
struct PersistentWorkspaceScope {
  PersistentWorkspaceScope();
  ~PersistentWorkspaceScope();
  bool prev;
};

int tc_debug_wgrad(long long* cycles, int* shapes, int max_ctas);

// diagnostics: the first B200_TC_OFFSET_GMAX entries of the b200_*_tc_image_offsets vector (see the header) for the
// images of a stand-alone call whose tensor-core workspace starts at tc_ws, or of one network of the fused step
void tc_single_image_offsets(const MlpShape& sh, TcNet net, int64_t rows, char* tc_ws, const char* ws, int64_t* out);
void tc_step_image_offsets(const MlpShape& ms, const MlpShape& as, const TcPlan& plan, bool atlas, const char* ws,
                           int64_t* out);
// the whole vector for b200_mlp_forward / backward(d, ..., rows, B200_PREC_TC, call_ws, ...), as byte offsets from
// `origin` (call_ws itself, or the start of a workspace that holds call_ws as a slice)
int tc_call_image_offsets(const B200MlpDesc* d, int64_t rows, const void* call_ws, const void* origin, int64_t* out);

}  // namespace b200
