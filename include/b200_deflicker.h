/* b200_deflicker.h — C ABI of libb200deflicker.so
 *
 * H100-native (sm_90a) replacement for the stage-1 neural-atlas hot path of
 * ChenyangLEI/All-In-One-Deflicker.  The reference has no FFI layer of its own: its operator
 * boundary for this path is the Python surface listed beside each entry point below (paths
 * relative to the reference root).  The Python mirror of that surface lives in
 * all-in-one-deflicker_b200/src/ and calls these functions through ctypes
 * (all-in-one-deflicker_b200/b200/_native.py); INTEGRATION.md shows the binding.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; the caller owns all memory
 *     (PyTorch allocates, the library borrows the pointers for the duration of the call / graph);
 *   - `stream` is a cudaStream_t passed as void*; all work is stream-ordered and CUDA-graph
 *     capturable: no allocation, no synchronisation, no host read-back inside any call;
 *   - return value 0 = success, otherwise a B200_ERR_* code; b200_last_error() returns a
 *     thread-local message; no exceptions cross the ABI;
 *   - one host thread per GPU / process drives the library (the reference's own model: one Python
 *     process per device); the small host-side caches (device tables, kernel attributes, the TMA
 *     descriptor encoder) are not synchronised;
 *   - floating point is fp32 in memory everywhere.  `precision` selects how the 256-wide Linear
 *     layers are contracted: B200_PREC_FP32 = CUDA-core FFMA (bit-for-bit an fp32 GEMM),
 *     B200_PREC_TC = wgmma tensor cores on a 2-term fp16 split of both operands (22-bit
 *     significands, fp32 accumulation in registers; DESIGN.md §numerics).
 */
#ifndef B200_DEFLICKER_H
#define B200_DEFLICKER_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_INVALID 1      /* bad argument (shape, null pointer, unsupported size)   */
#define B200_ERR_CUDA 2         /* a CUDA runtime call failed                               */
#define B200_ERR_WORKSPACE 3    /* workspace too small                                      */
#define B200_ERR_UNSUPPORTED 4  /* valid request this build cannot serve (e.g. no sm_90a)   */

#define B200_PREC_FP32 0
#define B200_PREC_TC 1

#define B200_MAX_LAYERS 16
#define B200_RECORD_FLOATS 16   /* floats per pixel record, see B200Video                    */

const char* b200_last_error(void);
int b200_version(void);
/* 1 if the current device is compute capability 9.x (wgmma path usable), else 0 */
int b200_device_supports_tc(void);

/* Diagnostics (no reference counterpart).  b200_launch_count: kernels this library has launched
 * (or captured into a CUDA graph) in this process.  b200_set_kernel_timer: record the two
 * cudaEvent_t around the launch site tagged `tag` (B200_TAG_*) on every following call, also
 * inside captured graphs; every tag has its own pair (all sites can be timed in one run); NULL
 * events switch that site off, (NULL, NULL, 0) switches every site off. */
#define B200_TAG_MAP_FWD 1
#define B200_TAG_MAP_BWD 2
#define B200_TAG_ATLAS_FWD 3
#define B200_TAG_ATLAS_BWD 4
#define B200_TAG_WGRAD 5
#define B200_TAG_ADAM 6
long long b200_launch_count(void);
/* Diagnostics: cycles each CTA of the LAST weight-gradient launch of the training step was busy, and the shape
 * (dZ columns, input columns, number of CTAs sharing the GEMM) of its work item; HOST arrays of max_ctas and
 * 3 * max_ctas entries; returns the number of CTAs or -1.  Synchronises the device. */
int b200_debug_wgrad(long long* cycles_host, int32_t* shapes_host, int32_t max_ctas);
int b200_set_kernel_timer(void* ev_start, void* ev_stop, int tag);
/* The tensor-core job tables that calls on a persistent workspace cache (the fused step, pre-training, the
 * segmentation step and render) are keyed by the workspace, parameter and gradient pointers and the row geometry, and
 * are held until released.  b200_tc_release_tables frees the current device's entries whose parameters lie in
 * [params, params + bytes): the owner of that parameter buffer calls it when it is done, after the last replay of any
 * CUDA graph captured over those calls.  Returns the number freed.  b200_tc_cached_tables: entries held now. */
int b200_tc_release_tables(const void* params, int64_t bytes);
int b200_tc_cached_tables(void);

/* ------------------------------------------------------------------------------------------
 * IMLP  — replaces  src/models/stage_1/implicit_neural_networks.py:15-81  (class IMLP)
 * ------------------------------------------------------------------------------------------ */
typedef struct B200MlpDesc {
  int32_t input_dim;       /* IMLP(input_dim=...)                                            */
  int32_t output_dim;      /* IMLP(output_dim=...)                                           */
  int32_t hidden_dim;      /* must be 256 for B200_PREC_TC                                   */
  int32_t num_layers;      /* includes the output layer, <= B200_MAX_LAYERS                  */
  int32_t pe_freqs;        /* positional_dim when use_positional else 0                      */
  uint32_t skip_mask;      /* bit i set  <=>  i in skip_layers                               */
  int32_t use_tanh;        /* tanh on the output                                             */
  int32_t reserved;
} B200MlpDesc;

/* Flat parameter layout of one network: for each layer the weight (out x in, row major — the
 * layout of nn.Linear.weight, `hidden.{i}.weight`) followed by the bias (`hidden.{i}.bias`),
 * every tensor starting at a multiple of 4 floats (gaps are zero and are never read as
 * parameters).  Fills w_off[i], b_off[i] (float offsets) and returns the padded float count, or
 * -1 on an invalid descriptor. */
int64_t b200_mlp_layout(const B200MlpDesc* d, int64_t* w_off, int64_t* b_off);

/* bytes of scratch b200_mlp_forward / backward need for `rows` rows (training!=0 keeps the
 * activations for a following backward) */
int64_t b200_mlp_workspace_bytes(const B200MlpDesc* d, int64_t rows, int training);

/* y[rows, output_dim] = IMLP(x[rows, input_dim])         (implicit_neural_networks.py:62-81) */
int b200_mlp_forward(const B200MlpDesc* d, const float* params, const float* x, float* y,
                     int64_t rows, int training, int precision, void* ws, int64_t ws_bytes,
                     void* stream);

/* Gradients of a forward(training=1) that used the same ws and the same x: dparams += dL/dparams
 * (flat layout, caller zeroes), dx = dL/dx (may be NULL; needs rows*enc*4 extra workspace bytes
 * when the network has a positional encoding).  Skip-concatenated inputs receive no input gradient
 * (`x.detach().clone()`, implicit_neural_networks.py:69). */
int b200_mlp_backward(const B200MlpDesc* d, const float* params, const float* x, const float* dy,
                      float* dparams, float* dx, int64_t rows, int precision, void* ws,
                      int64_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Device-resident video — replaces the eight CPU tensors of
 * src/models/stage_1/unwrap_utils.py:105-163 (load_input_data_single) and the (3,N) int64 index
 * table of get_tuples (unwrap_utils.py:166-173, recomputed arithmetically from the index).
 * ------------------------------------------------------------------------------------------ */
typedef struct B200Video {
  /* frame-major pixel records [t_end - t_begin][H][W][16] fp32:
   *   0..2 rgb | 3..5 d/dx rgb | 6..8 d/dy rgb | 9,10 forward flow | 11,12 backward flow |
   *   13 forward mask | 14 backward mask | 15 unused                                         */
  const float* records;
  /* validity bitmaps of the WHOLE video (bit n = pixel n of the index table), replicated on
   * every rank so the global flow-row counts need no collective                              */
  const uint32_t* mask_fwd_bits;
  const uint32_t* mask_bwd_bits;
  int32_t H, W, T;          /* full video                                                     */
  int32_t t_begin, t_end;   /* frames resident on this device                                 */
  int32_t reserved;
} B200Video;

/* Repack reference-layout device tensors (frames, dx, dy: (H,W,3,T); flows: (H,W,2,T,1);
 * masks: (H,W,T,1); T innermost) into records for frames [t_begin, t_end) and into the two
 * whole-video bitmaps (each ceil(H*W*T/32) words). */
int b200_video_pack(const float* frames, const float* frames_dx, const float* frames_dy,
                    const float* flow_fwd, const float* flow_bwd, const float* mask_fwd,
                    const float* mask_bwd, int32_t H, int32_t W, int32_t T, int32_t t_begin,
                    int32_t t_end, float* records, uint32_t* mask_fwd_bits,
                    uint32_t* mask_bwd_bits, void* stream);

/* ------------------------------------------------------------------------------------------
 * One loop trip — replaces src/stage1_neural_atlas.py:159-227 + loss.backward() (:230):
 * sampling/gather, 7 mapping + 3 atlas evaluations, RGB / gradient / rigidity / flow losses
 * (src/models/stage_1/loss_utils.py:134-170,227-278,299-356) and all parameter gradients.
 * ------------------------------------------------------------------------------------------ */
typedef struct B200AtlasConfig {
  int32_t batch;             /* samples_batch (global)                                        */
  int32_t with_global;       /* include_global_rigidity_loss && i <= stop_global_rigidity     */
  int32_t precision;         /* B200_PREC_*                                                   */
  int32_t resx;              /* width  — the gradient loss normalises by resx (loss_utils.py:138);
                                <= 0 means the video's width W (the rest normalises by max(W, H)) */
  float uv_mapping_scale;
  float derivative_amount;
  float global_derivative_amount;
  float rgb_coeff, gradient_coeff, rigidity_coeff, global_rigidity_coeff, flow_coeff;
} B200AtlasConfig;

/* loss vector written by b200_atlas_loss_grad (this rank's partial sums, already normalised by
 * the GLOBAL batch / flow counts, so a sum over ranks gives the reference's values):
 *   0 total  1 rgb  2 gradient  3 rigidity  4 global rigidity  5 flow  6 n_fwd  7 n_bwd        */
#define B200_LOSS_FLOATS 8

int64_t b200_atlas_param_floats(void);   /* mapping block followed by atlas block, padded */
int64_t b200_atlas_workspace_bytes(const B200AtlasConfig* cfg);

/* The mapping network of the script is a config choice (src/stage1_neural_atlas.py:112-119):
 * use_positional_encoding_mapping1 puts a positional encoding of number_of_positional_encoding_mapping1
 * frequencies in front of it.  Every atlas-step entry point has a `_for` form that takes the mapping
 * descriptor: 3 -> 256 x 4 -> 2 (6 layers, no skips, tanh), on the raw (x, y, t) (pe_freqs = 0) or on
 * their encoding (pe_freqs 1..10; b200_mlp_tc_architecture 1 or 4).  The forms without `_for` are the
 * default mapping (pe_freqs = 0).  The parameter buffer is the mapping block (b200_mlp_layout of
 * `mapping`) followed by the atlas block; b200_atlas_param_floats_for returns -1 for another mapping. */
int64_t b200_atlas_param_floats_for(const B200MlpDesc* mapping);
int64_t b200_atlas_workspace_bytes_for(const B200AtlasConfig* cfg, const B200MlpDesc* mapping);

/* indices: `batch` int64 pixel-table indices n -> (x = n % W, y = (n / W) % H, t = n / (H*W)),
 * identical on every rank; rows whose frame is not resident are skipped.  grads (same layout
 * as params) and losses are overwritten. */
int b200_atlas_loss_grad(const B200AtlasConfig* cfg, const B200Video* video,
                         const int64_t* indices, const float* params, float* grads,
                         float* losses, void* ws, int64_t ws_bytes, void* stream);
int b200_atlas_loss_grad_for(const B200AtlasConfig* cfg, const B200MlpDesc* mapping,
                             const B200Video* video, const int64_t* indices, const float* params,
                             float* grads, float* losses, void* ws, int64_t ws_bytes, void* stream);

/* Test / debugging aid: byte offsets (from `ws`) of the step's intermediate buffers inside the
 * workspace, for the configuration `cfg`: [0] counters (int32: n_local, n_fwd, n_bwd, ...),
 * [1] local sample list, [2] coordinate rows x_map [groups][cap][4], [3] gathered targets
 * [cap][12], [4] d_uv, [5] d_y, [6] mapping output uv [groups][cap][2], [7] atlas output
 * [3][cap][3].  cap = batch rounded up to 128. */
int b200_atlas_workspace_offsets(const B200AtlasConfig* cfg, const void* ws, int64_t* offsets);
int b200_atlas_workspace_offsets_for(const B200AtlasConfig* cfg, const B200MlpDesc* mapping,
                                     const void* ws, int64_t* offsets);

/* Test / debugging aid: where the tensor-core path (B200_PREC_TC) keeps the operand images of one
 * network inside a workspace, computed by the planning functions its launches use.  out receives
 * B200_TC_OFFSET_FLOATS int64:
 *   [0..7]   byte offsets from `ws` of: forward weight items, dgrad (W^T) weight items, forward
 *            constants, activation images, dZ images, positional-encoding image, output-layer dZ
 *            image, ReLU flag words (-1 where the network has no such buffer)
 *   [8..11]  bytes from one activation / dZ slot to the next, from the hi to the lo term of those
 *            images, from the hi to the lo term of the 64-wide images; rows of the images
 *   [12..27] byte offset of layer l's forward weight items from [0]
 *   [28..43] number of 64-wide k chunks (4 items each) of layer l's forward weight items
 *   [44..59] byte offset of layer l's dgrad weight items from [1]
 *   [60]     byte offset of the two int32 gmax words the backward took its gradient scales from
 *            ([0] atlas-shaped networks, [1] mappings)
 * b200_mlp_tc_image_offsets: the workspace of b200_mlp_forward / backward(d, ..., rows, B200_PREC_TC,
 * ws, ...).  b200_atlas_tc_image_offsets_for: the workspace of b200_atlas_loss_grad_for(cfg, mapping,
 * ..., ws, ...), net 0 = the mapping, 1 = the atlas. */
#define B200_TC_OFFSET_GMAX 60
#define B200_TC_OFFSET_FLOATS 61
int b200_mlp_tc_image_offsets(const B200MlpDesc* d, int64_t rows, const void* ws, int64_t* out);
int b200_atlas_tc_image_offsets_for(const B200AtlasConfig* cfg, const B200MlpDesc* mapping,
                                    const void* ws, int32_t net, int64_t* out);
/* The same vector for one network of a b200_seg_loss_grad(cfg, ..., ws, ...) workspace (declared
 * with B200SegConfig below): net 0 = mapping1, 1 = mapping2, 2 = alpha, 3 = atlas.  Each network's
 * images lie in its own slice of `ws`, planned for the rows the trip passes it (groups x cap, cap =
 * batch rounded up to 128: 9 or, without the global rigidity term, 7 groups for the mappings, 5
 * for alpha, 6 for the atlas); [11] is that row count.  Offsets are from `ws`.  A network the
 * configuration runs on the fp32 kernels has no images: the call fails and says so. */
struct B200SegConfig;
int b200_seg_tc_image_offsets(const struct B200SegConfig* cfg, const void* ws, int32_t net, int64_t* out);

/* One pre_train_mapping step (src/models/stage_1/unwrap_utils.py:182-195): rows ys / columns
 * xs (int64[batch]) of frame `frame`; gradients of the mapping block only; loss -> losses[0]. */
int b200_pretrain_loss_grad(const B200AtlasConfig* cfg, int32_t larger_dim, int32_t T,
                            int32_t frame, const int64_t* ys, const int64_t* xs,
                            const float* params, float* grads, float* losses, void* ws,
                            int64_t ws_bytes, void* stream);
int b200_pretrain_loss_grad_for(const B200AtlasConfig* cfg, const B200MlpDesc* mapping,
                                int32_t larger_dim, int32_t T, int32_t frame, const int64_t* ys,
                                const int64_t* xs, const float* params, float* grads,
                                float* losses, void* ws, int64_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Input producer on the device — replaces the per-frame / per-pair arithmetic of
 *   load_input_data_single   src/models/stage_1/unwrap_utils.py:105-163
 *   resize_flow              :33-38   (cv2.resize INTER_LINEAR + the swapped scale factors)
 *   compute_consistency      :10-23   (cv2.remap bilinear, zero border; mask = error < 1.0)
 * writing B200Video.records / bitmaps directly (no (H,W,.,T) host tensors).  Bit-exact with the
 * reference's tensors for flows that are not smaller than the working resolution (down-scaling or
 * equal size; an up-scaling flow is refused with B200_ERR_INVALID: resize it on the host first).
 * `records` and the bitmaps must be zero-initialised once (slots of missing partners stay 0).
 * ------------------------------------------------------------------------------------------ */
/* frame: decoded + resized frame (H, W, 3) fp32 in [0,1]; frame_records: records of that frame */
int b200_producer_frame(const float* frame, int32_t H, int32_t W, float* frame_records,
                        void* stream);
int64_t b200_producer_scratch_floats(int32_t H, int32_t W);
/* flow12 / flow21: the two RAFT flows of the frame pair (first_frame, first_frame + 1), (h, w, 2)
 * fp32 as stored in <vid>_flow/{a}_{b}.npy.  (H, W, T, t_begin, t_end) as in B200Video; records =
 * the resident records (NULL on a rank that holds neither frame: only the whole-video bitmaps,
 * replicated on every rank, are updated).  filter = filter_optical_flow. */
int b200_producer_flow_pair(const float* flow12, const float* flow21, int32_t h, int32_t w,
                            int32_t H, int32_t W, int32_t T, int32_t t_begin, int32_t t_end,
                            float* records, uint32_t* mask_fwd_bits, uint32_t* mask_bwd_bits,
                            int32_t first_frame, int32_t filter, float* scratch, void* stream);

/* ------------------------------------------------------------------------------------------
 * Stage-2 frame plumbing on the device — replaces, per frame, the host arithmetic of
 *   load_image x2 + InputPadder.pad + torch.cat          src/models/utils.py, neural_filter_and_refinement.py:59-62
 *   cv2.resize(tensor2img(t), org_size) + save_img       :69-72
 * 8-bit images in, 8-bit images out.  cv2.resize is restated as OpenCV's own INTER_LINEAR code computes it
 * (oracle/stage2_io_oracle.py resize_linear_f64 / resize_linear_f32, pinned against cv2.resize with its IPP
 * back end switched off; where OpenCV dispatches float images to IPP the host results differ in the last bits).
 * ------------------------------------------------------------------------------------------ */
/* out [1][6][Hp][Wp] fp32: channels 0-2 = content / 255, channels 3-5 = atlas / 255 resized (Hs, Ws) -> (Hc, Wc),
 * both replicate-padded to Hp = Hc rounded up to 32 (all rows at the bottom) and Wp = Wc rounded up to 32 (pad // 2
 * columns on the left, the rest on the right).  content (Hc, Wc, Cc) and atlas (Hs, Ws, Cs) are contiguous uint8 HWC
 * device images with 1 (grey, repeated), 3 or 4 (4th dropped) channels.  The division and the resize are float64 with
 * fp32 weights, rounded to fp32 once, as load_image computes them. */
int b200_stage2_pack_input(const uint8_t* content, int32_t Hc, int32_t Wc, int32_t Cc,
                           const uint8_t* atlas, int32_t Hs, int32_t Ws, int32_t Cs, float* out,
                           int32_t Hp, int32_t Wp, void* stream);
/* src: 3 fp32 planes (Hp, Wp), plane_stride floats apart (a channel slice of a padded NCHW tensor), squeezed to
 * (H, W) by the fp32 resize exactly as the reference squeezes the padded tensor, then
 * clip(v * 255, 0, 255) truncated to uint8 (NaN gives 0), RGB -> BGR, written as rows of 3 W bytes at
 * dst + dst_offset + y * dst_row_stride; no other byte of dst is touched. */
int b200_stage2_emit(const float* src, int64_t plane_stride, int32_t Hp, int32_t Wp, uint8_t* dst,
                     int64_t dst_offset, int64_t dst_row_stride, int32_t H, int32_t W, void* stream);

/* ------------------------------------------------------------------------------------------
 * PNG encoding of an 8-bit BGR image, byte for byte the file
 *   cv2.imwrite(path, img, [cv2.IMWRITE_PNG_COMPRESSION, 0])        save_img, src/models/utils.py
 * writes (libpng's adaptive row filters on RGB, zlib stored blocks).  What depends on the pixels — the row filters,
 * the filtered bytes, the Adler-32 and the IDAT CRC-32s — is computed on the device; what depends on (H, W) only —
 * zlib header, stored-block lengths, IDAT chunk lengths, the bytes before the first and after the last IDAT chunk —
 * is a plan the caller builds once per shape from the layout of the writer's file of any image of that shape.
 * ------------------------------------------------------------------------------------------ */
#define B200_PNG_PLAN_MAGIC 0x504e4731     /* "PNG1" */
#define B200_PNG_MAX_CHUNK 32768           /* longest IDAT chunk a plan may have (libpng writes 8192)      */
#define B200_PNG_MAX_PREFIX 4096           /* longest run of bytes before the first / after the last IDAT  */
#define B200_PNG_MAX_RAW (1ll << 30)       /* H (3 W + 1): filtered bytes of one image                     */
/* Header of a plan; the tables follow it in the same buffer at the byte offsets *_at.  The plan is plain bytes: the
 * caller keeps the host copy (b200_png_encode reads its header) and uploads the whole of it once. */
typedef struct B200PngPlan {
  int32_t magic;                   /* B200_PNG_PLAN_MAGIC                                           */
  int32_t H, W;
  int32_t n_blocks, n_chunks;      /* stored deflate blocks, IDAT chunks                            */
  int32_t prefix_bytes, suffix_bytes;
  int32_t max_chunk;               /* longest IDAT chunk                                            */
  int64_t raw_bytes;               /* H (3 W + 1): filtered rows, each led by its filter byte       */
  int64_t zlib_bytes;              /* 2 + 5 n_blocks + raw_bytes + 4                                */
  int64_t file_bytes;              /* prefix + 12 n_chunks + zlib_bytes + suffix                    */
  int64_t plan_bytes;              /* header and tables                                             */
  int64_t block_raw_at;            /* uint32 [n_blocks + 1]: raw offset of each block, then raw_bytes */
  int64_t chunk_z_at;              /* uint32 [n_chunks + 1]: zlib offset of each chunk, then zlib_bytes */
  int64_t prefix_at, suffix_at;    /* the bytes before the first IDAT chunk / after the last        */
  uint8_t zlib_header[8];          /* CMF, FLG; the rest 0                                          */
} B200PngPlan;
/* bytes of a plan with these table sizes; -1 (message) when a size is out of range */
int64_t b200_png_plan_bytes(int32_t n_blocks, int32_t n_chunks, int32_t prefix_bytes, int32_t suffix_bytes);
/* Host only.  Validates a layout and writes the plan into `plan` (host memory, plan_capacity bytes):
 * zlib_header[2]; block_heads[b] the stored blocks' first bytes (0, the last 1: BFINAL, BTYPE 00) and block_lens[b]
 * their lengths (<= 65535, summing to H (3 W + 1)); chunk_lens[c] the IDAT lengths (1 .. B200_PNG_MAX_CHUNK,
 * summing to the zlib stream's length); prefix = signature, IHDR (8-bit RGB, H x W, not interlaced), any other
 * chunk before the first IDAT; suffix = the chunks after the last, ending with IEND. */
int b200_png_plan(int32_t H, int32_t W, const uint8_t* zlib_header, const uint8_t* block_heads,
                  const int32_t* block_lens, int32_t n_blocks, const int32_t* chunk_lens, int32_t n_chunks,
                  const uint8_t* prefix, int32_t prefix_bytes, const uint8_t* suffix, int32_t suffix_bytes,
                  void* plan, int64_t plan_capacity);
/* device workspace of one encode (the filtered rows and per-row Adler-32 sums); -1 (message) for a bad size */
int64_t b200_png_workspace_bytes(int32_t H, int32_t W);
/* Encodes the contiguous uint8 BGR device image (plan->H, plan->W, 3) into out[0, plan->file_bytes).
 * plan = the host plan, plan_device = its upload (8-byte aligned).  Two launches, no allocation, no
 * synchronisation; workspace_bytes and out_capacity are checked against the plan. */
int b200_png_encode(const B200PngPlan* plan, const void* plan_device, const uint8_t* image, void* workspace,
                    int64_t workspace_bytes, uint8_t* out, int64_t out_capacity, void* stream);

/* ------------------------------------------------------------------------------------------
 * Data-parallel optimiser step (frame-sharded loop, SURVEY.md §8e): reduce-scatter of the partial
 * [gradients || 8 losses] buffers + Adam + all-gather of the new parameters in ONE kernel over
 * NVLink peer memory.  Replaces  torch.distributed.all_reduce + optimizer.step()  of a data-parallel
 * port of src/stage1_neural_atlas.py:229-231.  Every rank calls it once per iteration with the same
 * arguments; the buffers are symmetric allocations (same size on every rank, peer-mapped):
 *   partials[j]  rank j's flat buffer of n_total floats (gradients then the loss vector): read by all
 *                ranks; on return its last (n_total - n_params) floats hold the global loss sums
 *                (the one place the call writes through this pointer)
 *   params[j]    rank j's flat parameters: on return identical on all ranks
 *   flags[j]     rank j's 2*world uint64 flags (zero-initialised once, then owned by this call)
 * exp_avg / exp_avg_sq are local; a rank maintains only the moments of its slice
 * [rank * ceil(total4 / world), ...) in float4 units (b200_dp_slice).  `step` as in b200_adam_step;
 * `epoch` is a device counter private to this call (zero-initialised).  Graph-capturable; the ranks
 * must run the call concurrently (it waits on peer flags).
 * ------------------------------------------------------------------------------------------ */
#define B200_MAX_RANKS 16
typedef struct B200DpComm {
  int32_t world, rank;
  const float* partials[B200_MAX_RANKS];
  float* params[B200_MAX_RANKS];
  unsigned long long* flags[B200_MAX_RANKS];
} B200DpComm;
int b200_dp_adam_step(const B200DpComm* comm, float* exp_avg, float* exp_avg_sq, int64_t n_params,
                      int64_t n_total, double lr, double beta1, double beta2, double eps,
                      int64_t* step, unsigned long long* epoch, void* stream);
/* first float and number of floats of rank's slice of a buffer of n_total floats */
int b200_dp_slice(int32_t world, int32_t rank, int64_t n_total, int64_t* begin, int64_t* count);

/* ------------------------------------------------------------------------------------------
 * Stand-alone loss heads — the arithmetic of the reference's three loss FUNCTIONS
 *   get_gradient_loss_single  src/models/stage_1/loss_utils.py:134-170
 *   get_rigidity_loss         src/models/stage_1/loss_utils.py:227-278
 *   get_optical_flow_loss     src/models/stage_1/loss_utils.py:299-322 (one flow direction per call)
 * for callers that keep the reference's function-level structure (all-in-one-deflicker_b200/src/
 * models/stage_1/loss_utils.py wraps them as autograd Functions).  Each call writes the scalar the
 * reference function returns (*loss, a mean) and the gradient of that scalar with respect to every
 * network output it consumes.  Inputs are the *network outputs* (rgb = (atlas+1)/2, uv = mapping);
 * evaluating the networks stays with the caller's IMLP objects.  rows n; all arrays row-major.
 * ------------------------------------------------------------------------------------------ */
/* rgb, rgb_xp, rgb_yp, dx_gt, dy_gt: [n][3]; d_*: [n][3] */
int b200_gradient_loss_head(const float* rgb, const float* rgb_xp, const float* rgb_yp,
                            const float* dx_gt, const float* dy_gt, int64_t n, float* loss,
                            float* d_rgb, float* d_rgb_xp, float* d_rgb_yp, void* stream);
/* uv: [n][2]; uv_p: [2n][2] = mapping at (x, y-d, t) for all rows, then at (x-d, y, t) (the
 * concatenation order of loss_utils.py:230-233); per_sample (optional, [n]) receives the
 * un-averaged values (`return_all=True`) */
int b200_rigidity_loss_head(const float* uv, const float* uv_p, int64_t n, float resx,
                            float uv_mapping_scale, float derivative_amount, float* per_sample,
                            float* loss, float* d_uv, float* d_uv_p, void* stream);
/* uv_rel, uv_match: [n][2] (rows with a valid flow only); n == 0 writes NaN like torch's mean */
int b200_flow_loss_head(const float* uv_rel, const float* uv_match, int64_t n, float resx,
                        float uv_mapping_scale, float* loss, float* d_uv_rel, float* d_uv_match,
                        void* stream);
/* the use_alpha=True form (loss_utils.py:316-318, segmentation variant): mean_rows w * ||.|| * resx /
 * (2 uv_mapping_scale) with per-row weights w [n] (alpha or 1 - alpha of the row's sample); d_w = dL/dw */
int b200_flow_loss_head_weighted(const float* uv_rel, const float* uv_match, const float* w,
                                 int64_t n, float resx, float uv_mapping_scale, float* loss,
                                 float* d_uv_rel, float* d_uv_match, float* d_w, void* stream);

/* ------------------------------------------------------------------------------------------
 * Optimiser — replaces torch.optim.Adam.step() (src/stage1_neural_atlas.py:132-134,231) on a
 * flat buffer.  `step` is a device int64 counter (steps already taken); it is incremented by
 * the kernel so the call can sit inside a replayed CUDA graph.  lr/betas/eps are doubles because
 * torch derives 1-beta and the bias corrections from Python floats.  grad_scale multiplies the
 * gradient first (1/world for an averaged all-reduce; 1.0 otherwise).
 * ------------------------------------------------------------------------------------------ */
int b200_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                   int64_t n, double lr, double beta1, double beta2, double eps, float grad_scale,
                   int64_t* step, void* stream);

/* ------------------------------------------------------------------------------------------
 * Render — replaces the reconstruction loop of src/models/stage_1/evaluate.py:640-666,733:
 * rgb[(y*W + x)*3 + c] of frame f for pixels [pix_begin, pix_end); also u8 = trunc(rgb * 255)
 * when rgb_u8 != NULL.
 * ------------------------------------------------------------------------------------------ */
int64_t b200_render_workspace_bytes(int64_t pixels);
int b200_render(const float* params, int32_t H, int32_t W, int32_t T, int32_t frame,
                int64_t pix_begin, int64_t pix_end, float* rgb, uint8_t* rgb_u8, int precision,
                void* ws, int64_t ws_bytes, void* stream);
/* the same with the mapping of b200_atlas_param_floats_for */
int64_t b200_render_workspace_bytes_for(const B200MlpDesc* mapping, int64_t pixels);
int b200_render_for(const B200MlpDesc* mapping, const float* params, int32_t H, int32_t W,
                    int32_t T, int32_t frame, int64_t pix_begin, int64_t pix_end, float* rgb,
                    uint8_t* rgb_u8, int precision, void* ws, int64_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Segmentation variant of the loop — replaces src/stage1_neural_atlas_seg.py:207-315 +
 * loss.backward(): foreground / background mapping networks, alpha network, one atlas network
 * sampled in two quadrants (uv*0.5 +- 0.5); two-layer gradient loss (loss_utils.py:173-224),
 * rigidity of both mappings (:227-278), alpha-weighted flow losses (:299-322, use_alpha=True),
 * alpha flow loss (:385-408), bootstrapping BCE and sparsity (seg script :249-307).
 * The four networks may have any IMLP shape; with precision == B200_PREC_TC each network whose
 * shape has tensor-core kernels (b200_mlp_tc_architecture != 0) uses them, the others the fp32
 * kernels.  The video may be the whole clip or a frame shard (t_begin, t_end with the
 * whole-video bitmaps, as for b200_atlas_loss_grad): a rank evaluates its resident samples only
 * (the tensor-core launches visit only the tiles that hold them), normalised by the GLOBAL batch
 * and flow counts, so that one SUM over the ranks of [grads || losses] is the unsharded trip.
 * ------------------------------------------------------------------------------------------ */
typedef struct B200SegConfig {
  int32_t batch;             /* samples_batch                                                  */
  int32_t with_global;       /* include_global_rigidity_loss && i <= stop_global_rigidity      */
  int32_t precision;         /* B200_PREC_*                                                    */
  int32_t resx;              /* width (gradient-loss normalisation); <= 0 means the video's
                                width W, as for B200AtlasConfig::resx                           */
  float uv_mapping_scale;
  float derivative_amount;
  float global_derivative_amount;   /* global_rigidity_derivative_amount_fg == _bg (both 100 in the
                                       reference's config; different values are not supported)  */
  float rgb_coeff, gradient_coeff, rigidity_coeff;
  float global_rigidity_coeff_fg, global_rigidity_coeff_bg;
  float flow_coeff;          /* optical_flow_coeff                                             */
  float alpha_flow_factor, sparsity_coeff;
  float bootstrapping_factor;/* alpha_bootstrapping_factor, 0 after stop_bootstrapping_iteration */
  B200MlpDesc mapping1, mapping2, alpha, atlas;
} B200SegConfig;

/* loss vector of b200_seg_loss_grad:
 *   0 total  1 rgb  2 gradient  3 sparsity  4 rigidity1  5 rigidity2  6 global rigidity1
 *   7 global rigidity2  8 flow1  9 flow2  10 flow alpha  11 bootstrapping  12 n_fwd  13 n_bwd
 * On a frame shard 0-11 are this rank's share; 12, 13 are the whole batch's counts on every rank
 * (world * count after a SUM over ranks).  The flow terms are NaN on every rank when a count is 0. */
#define B200_SEG_LOSS_FLOATS 16

/* Which tensor-core kernels serve a network shape: 1 = mapping-shaped (3 -> 256 x {2,4} -> 2, no
 * encoding: both mappings of the scripts), 2 = the atlas network (2 -> PE 10 -> 256 x 6 -> 3, skips 4
 * and 7), 3 = the alpha network of the segmentation variant (3 -> PE 5 -> 256 x 6 -> 1), 4 = a
 * position-encoded mapping (3 -> PE P -> 256 x {2,4} -> 2, P = 1..10, no skips: the mappings with
 * use_positional_encoding_mapping1/2), 0 = any other shape (fp32 kernels only), -1 = invalid
 * descriptor.  Codes 1 and 4 have no input gradient on the tensor cores. */
int b200_mlp_tc_architecture(const B200MlpDesc* d);

/* parameters / gradients / Adam moments are ONE flat buffer: the four networks in the order of
 * the script's optimiser groups (mapping1, mapping2, alpha, atlas), each in b200_mlp_layout.
 * Fills offsets[4] (floats) and returns the total, or -1. */
int64_t b200_seg_param_floats(const B200SegConfig* cfg, int64_t* offsets);
int64_t b200_seg_workspace_bytes(const B200SegConfig* cfg);

/* mask: the bootstrapping mask of the RESIDENT frames as [t_end - t_begin][H][W] fp32
 * (mask_frames[y, x, t] of load_input_data, unwrap_utils.py:40-72, frame-major; the whole [T][H][W]
 * mask when the whole video is resident).  grads and losses are overwritten. */
int b200_seg_loss_grad(const B200SegConfig* cfg, const B200Video* video, const float* mask,
                       const int64_t* indices, const float* params, float* grads, float* losses,
                       void* ws, int64_t ws_bytes, void* stream);

/* Test / debugging aid: byte offsets (from `ws`) of the intermediate buffers of b200_seg_loss_grad
 * inside its workspace, for the configuration `cfg` (host only, no launch).  out receives
 * B200_SEG_OFFSET_FLOATS int64, cap = batch rounded up to 128:
 *   [0] counters (int32, as in the atlas step)  [1] x_map [9][cap][4]  [2] targets [cap][12]
 *   [3] x3 [9][cap][3]  [4] xa [5][cap][3]  [5] xat [6][cap][2]  [6] uv1 [9][cap][2]
 *   [7] uv2 [9][cap][2]  [8] ar [5][cap]  [9] yat [6][cap][3]  [10] d_uv1  [11] d_uv2  [12] d_ar
 *   [13] d_yat  [14] d_xat (same shapes as the buffers they are the gradients of) */
#define B200_SEG_OFFSET_FLOATS 15
int b200_seg_workspace_offsets(const B200SegConfig* cfg, const void* ws, int64_t* out);

/* One pre_train_mapping step (unwrap_utils.py:182-195) for ANY mapping-shaped IMLP (3 -> 2):
 * gradients of that network (its own flat layout, overwritten); loss -> losses[0]. */
int64_t b200_mlp_pretrain_workspace_bytes(const B200MlpDesc* d, int32_t batch);
int b200_mlp_pretrain_loss_grad(const B200MlpDesc* d, int32_t batch, float uv_mapping_scale,
                                int32_t larger_dim, int32_t T, int32_t frame, const int64_t* ys,
                                const int64_t* xs, const float* params, float* grads,
                                float* losses, int precision, void* ws, int64_t ws_bytes,
                                void* stream);

/* Reconstruction of the seg variant (src/models/stage_1/evaluate.py:293-335): composite
 * rgb = rgb1*alpha + rgb2*(1-alpha) and alpha for pixels [pix_begin, pix_end) of frame f.
 * rgb [count][3], rgb_u8 (may be NULL), alpha [count] (may be NULL).  A frame outside [0, T) is
 * refused with B200_ERR_INVALID, as b200_render refuses it. */
int64_t b200_seg_render_workspace_bytes(const B200SegConfig* cfg, int64_t pixels);
int b200_seg_render(const B200SegConfig* cfg, const float* params, int32_t H, int32_t W, int32_t T,
                    int32_t frame, int64_t pix_begin, int64_t pix_end, float* rgb,
                    uint8_t* rgb_u8, float* alpha, void* ws, int64_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Evaluation maps of one frame — the per-pixel quantities of the reference's evaluation output
 * (src/models/stage_1/evaluate.py:640-708): uv of every pixel, its rigidity loss
 * (get_rigidity_loss(..., return_all=True), loss_utils.py:227-278) and its forward flow error
 * (get_optical_flow_loss_all, loss_utils.py:283-295; zero where the flow is invalid and for the
 * last frame).  `mapping` + `mapping_params`: one mapping network in its own flat layout.
 * Outputs for pixels [pix_begin, pix_end) of `frame` (each may be NULL): uv [count][2],
 * rigidity [count], flow_error [count].
 * ------------------------------------------------------------------------------------------ */
int64_t b200_eval_maps_workspace_bytes(const B200MlpDesc* mapping, int64_t pixels);
int b200_eval_maps(const B200MlpDesc* mapping, const float* mapping_params, const B200Video* video,
                   int32_t frame, int64_t pix_begin, int64_t pix_end, float derivative_amount,
                   float uv_mapping_scale, int precision, float* uv, float* rigidity,
                   float* flow_error, void* ws, int64_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Squared error of one rendered frame — the numerator of the evaluation's per-frame PSNR
 * (src/models/stage_1/evaluate.py:740-743) against the fp32 frame held in channels 0..2 of the
 * frame's resident records.  `rgb`: (H, W, 3) fp32 on the device; `*out` (device) receives the
 * float64 sum over the H*W*3 values of (rgb - record)^2.  The summation order depends on H*W only
 * (per-CTA partials, then one CTA; no atomics): bit-identical across calls, graph replays and
 * ranks, and graph-capturable.  A frame outside [t_begin, t_end) is refused with B200_ERR_INVALID,
 * a workspace below b200_frame_sse_workspace_bytes(H, W) with B200_ERR_WORKSPACE.
 * ------------------------------------------------------------------------------------------ */
int64_t b200_frame_sse_workspace_bytes(int32_t H, int32_t W);
int b200_frame_sse(const B200Video* video, int32_t frame, const float* rgb, double* out, void* ws,
                   int64_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Temporal warping error of frame pairs (no reference counterpart; the metric of
 * fast_blind_video_consistency that the paper scores deflickering with; DESIGN §4e).  For frames t
 * and t+1 (frame0, frame1: (H, W, 3) uint8 or uint16 HWC, decoded as v / 255 or v / 65535 in fp32)
 * and the pre-pass flows fwd = F (t -> t+1) and bwd = B (t+1 -> t), (Hf, Wf, 2) fp32 (x, y): at
 * every pixel p, q = p + F(p); p is in the mask when q lies in [0, W-1] x [0, H-1] and
 * |F + B~|^2 <= 0.01 (|F|^2 + |B~|^2) + 0.5, B~ = bilinear sample of B at q.  The pair's error is
 * the sum over the mask of sum_c (frame0(p, c) - bilinear sample of frame1 at q)^2.  Flows of
 * another size are first resized to (H, W) in the workspace (cv2.resize INTER_LINEAR arithmetic in
 * fp32), x scaled by W / Wf and y by H / Hf.
 * ------------------------------------------------------------------------------------------ */
#define B200_WARP_MAX_PAIRS 32
typedef struct {
  const void* frame0;     /* frame t   (H, W, 3), uint8 when bits == 8, uint16 when bits == 16 */
  const void* frame1;     /* frame t+1 (H, W, 3), the same type */
  const float* fwd;       /* F (Hf, Wf, 2), 8-byte aligned */
  const float* bwd;       /* B (Hf, Wf, 2), 8-byte aligned */
  int32_t H, W;           /* the frames' size: the resolution the pair is scored at */
  int32_t Hf, Wf;         /* the flows' size */
  int32_t bits;           /* 8 or 16 */
  int32_t reserved;
} B200WarpPair;
/* bytes of workspace a call on these pairs needs; -1 (message) for an invalid table */
int64_t b200_warp_error_workspace_bytes(const B200WarpPair* pairs_host, int32_t n);
/* Scores n (1..B200_WARP_MAX_PAIRS) pairs in one launch sequence.  sums [n][2] float64: the masked
 * squared-error sum and the mask's pixel count.  error (fp32) and mask (uint8), each NULL or one
 * value per pixel, pair after pair: error = the pixel's sum over c of the squared difference where q
 * lies in the frame (0 where it does not), mask = 1 in the mask.  The per-pixel arithmetic is
 * float64, the error is rounded to fp32 once, and sums[i][0] is the float64 sum of those fp32
 * values over the mask in an order that depends on H * W only (no atomics): bit-identical across
 * calls, graph replays, batch compositions and devices. */
int b200_warp_error(const B200WarpPair* pairs_host, int32_t n, double* sums, float* error, uint8_t* mask,
                    void* ws, int64_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Fidelity of frames to a reference (no reference counterpart; the partner of the warping error,
 * DESIGN §4f).  For a frame O ((H, W, 3) uint8 or uint16 HWC, decoded as v / 255 or v / 65535 in
 * fp32) and a reference R ((Hr, Wr, 3), its own bit depth; resized to (H, W) with cv2.resize
 * INTER_LINEAR arithmetic in fp32 when the sizes differ): per channel c and interior pixel p
 * (5 <= x < W - 5, 5 <= y < H - 5), with G the separable Gaussian window (sigma 1.5, radius 5),
 * mu_O = G*O, mu_R = G*R, var_O = G*O^2 - mu_O^2, var_R likewise, cov = G*(O R) - mu_O mu_R,
 * SSIM = (2 mu_O mu_R + C1)(2 cov + C2) / ((mu_O^2 + mu_R^2 + C1)(var_O + var_R + C2)),
 * C1 = 0.01^2, C2 = 0.03^2.  H and W must be at least 11.
 * ------------------------------------------------------------------------------------------ */
#define B200_FIDELITY_MAX_FRAMES 32
typedef struct {
  const void* frame;      /* O (H, W, 3), uint8 when bits == 8, uint16 when bits == 16 */
  const void* ref;        /* R (Hr, Wr, 3), uint8 when ref_bits == 8, uint16 when ref_bits == 16 */
  int32_t H, W;           /* O's size: the resolution the frame is scored at */
  int32_t Hr, Wr;         /* R's size */
  int32_t bits;           /* O's: 8 or 16 */
  int32_t ref_bits;       /* R's: 8 or 16 */
} B200FidelityFrame;
/* bytes of workspace a call on these frames needs; -1 (message) for an invalid table */
int64_t b200_fidelity_workspace_bytes(const B200FidelityFrame* frames_host, int32_t n);
/* Scores n (1..B200_FIDELITY_MAX_FRAMES) frame pairs in one launch sequence.  sums [n][2] float64:
 * the SSIM sum over the (H - 10)(W - 10) interior pixels and 3 channels, and the squared-error sum
 * over all H W 3 values.  ssim_map (fp32), NULL or H * W * 3 values per pair, pair after pair: the
 * SSIM of each interior pixel and channel rounded to fp32 once, NaN outside the interior.  The
 * arithmetic is float64 with one IEEE rounding per operation, and the sums' order depends on H and
 * W only (no atomics): bit-identical across calls, graph replays, batch compositions and devices.
 * Allocates nothing, does not synchronise, graph-capturable. */
int b200_fidelity(const B200FidelityFrame* frames_host, int32_t n, double* sums, float* ssim_map, void* ws,
                  int64_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Cross-fade of two renders of one frame (no reference counterpart; the seams of overlapping clips,
 * DESIGN §5).  For each of the n values: o = (float)((1 - w) (double)a + w (double)b), in float64
 * with one IEEE rounding per operation and no fma, rounded to fp32 once, so w = 0 gives a and
 * w = 1 gives b exactly (for finite values other than -0); u8 = (uint8_t)(int)((double)o * 255.0),
 * the conversion of the stage-1 renders.  `out` (fp32) or `u8` may be NULL, not both.  w must be
 * finite and in [0, 1].  Allocates nothing, does not synchronise, graph-capturable.
 * ------------------------------------------------------------------------------------------ */
int b200_blend_frames(const float* a, const float* b, int64_t n, double w, float* out, uint8_t* u8, void* stream);

/* ------------------------------------------------------------------------------------------
 * RAFT correlation — replaces CorrBlock (src/models/stage_1/core/corr.py:16-64) with an all-pairs pyramid, and
 * AlternateCorrBlock (corr.py:67-91) with the on-the-fly b200_corr_alt_* calls below, which take the place of the
 * reference's unshipped alt_cuda_corr extension.
 * fmaps: [dim][H8*W8] fp32 (batch 1).  pyramid: level 0 [H8*W8][H8][W8], then 3 avg-pooled levels,
 * b200_corr_pyramid_floats() floats in total.
 * The *_batch forms take B pairs: fmaps [B][dim][H8*W8], pyramids [B][b200_corr_pyramid_floats(H8, W8)], coords
 * [B][2][H8][W8], outputs [B][4*(2r+1)^2][H8][W8].  Every sample's bits equal those of the single-pair call on it;
 * the single-pair calls are their B = 1 case (and refuse any other batch).  Lookups run the batch in one launch.
 * ------------------------------------------------------------------------------------------ */
int64_t b200_corr_pyramid_floats(int32_t H8, int32_t W8);
int b200_corr_build(const float* fmap1, const float* fmap2, int32_t dim, int32_t H8, int32_t W8,
                    float* pyramid, void* stream);
int b200_corr_build_batch(const float* fmap1, const float* fmap2, int32_t batch, int32_t dim, int32_t H8, int32_t W8,
                          float* pyramid, void* stream);
/* levels 1..3 from level 0 (2x2 average pooling over the target image, corr.py:22-25); called by both builders */
int b200_corr_pool_levels(float* pyramid, int32_t H8, int32_t W8, void* stream);
int b200_corr_pool_levels_batch(float* pyramid, int32_t batch, int32_t H8, int32_t W8, void* stream);
/* Tensor-core builder: level 0 on wgmma with both feature maps split into (hi, lo) fp16 pairs (3 products per
 * element, fp32 accumulation: fp32-grade like the reference's fp32 matmul), operands fed by TMA; then the pooling.
 * workspace: b200_corr_build_tc_workspace_bytes(dim, H8, W8) bytes.  The batched form builds the samples one after
 * the other in the same workspace: b200_corr_build_tc_batch_workspace_bytes(batch, dim, H8, W8) bytes. */
int64_t b200_corr_build_tc_workspace_bytes(int32_t dim, int32_t H8, int32_t W8);
int b200_corr_build_tc(const float* fmap1, const float* fmap2, int32_t dim, int32_t H8, int32_t W8, float* pyramid,
                       void* workspace, int64_t workspace_bytes, void* stream);
int64_t b200_corr_build_tc_batch_workspace_bytes(int32_t batch, int32_t dim, int32_t H8, int32_t W8);
int b200_corr_build_tc_batch(const float* fmap1, const float* fmap2, int32_t batch, int32_t dim, int32_t H8, int32_t W8,
                             float* pyramid, void* workspace, int64_t workspace_bytes, void* stream);
/* CorrBlock.__call__ (corr.py:33-54): coords [1][2][H8][W8] (x, y) -> out [1][4*(2r+1)^2][H8][W8]; radius 1..8 */
int b200_corr_lookup(const float* pyramid, const float* coords, float* out, int32_t batch,
                     int32_t H8, int32_t W8, int32_t radius, void* stream);
int b200_corr_lookup_batch(const float* pyramid, const float* coords, float* out, int32_t batch,
                           int32_t H8, int32_t W8, int32_t radius, void* stream);
/* On-the-fly correlation (AlternateCorrBlock): no all-pairs volume.  The state holds fmap1 and fmap2's four 2x2
 * average-pooled levels, pixel-major ([pixels][dim]): b200_corr_alt_floats(dim, H8, W8) floats (-1 for a geometry
 * the kernels do not take: dim a positive multiple of 16, H8, W8 >= 8), 16-byte aligned, owned by the caller.
 * The lookup forms each window's dot products / sqrt(dim) when it is looked up and returns what b200_corr_lookup
 * returns on the pyramid of the same fmaps, up to fp32 rounding (layout, taps, padding, NaN rules are the same);
 * batch 1, radius 1..8.  Both calls are stream-ordered, allocate nothing and can be captured in a CUDA graph.
 * The *_batch forms take B pairs with states [B][b200_corr_alt_floats(dim, H8, W8)], one launch per kernel. */
int64_t b200_corr_alt_floats(int32_t dim, int32_t H8, int32_t W8);
int b200_corr_alt_build(const float* fmap1, const float* fmap2, int32_t dim, int32_t H8, int32_t W8, float* state,
                        void* stream);
int b200_corr_alt_lookup(const float* state, const float* coords, float* out, int32_t dim, int32_t batch, int32_t H8,
                         int32_t W8, int32_t radius, void* stream);
int b200_corr_alt_build_batch(const float* fmap1, const float* fmap2, int32_t batch, int32_t dim, int32_t H8, int32_t W8,
                              float* state, void* stream);
int b200_corr_alt_lookup_batch(const float* state, const float* coords, float* out, int32_t dim, int32_t batch, int32_t H8,
                               int32_t W8, int32_t radius, void* stream);

/* ------------------------------------------------------------------------------------------
 * Convolution and image operators of the RAFT update block (core/update.py:6-136) and of the
 * stage-2 networks (src/models/network_filter.py:8-107, src/models/network_local.py:7-188).
 * NCHW fp32 tensors; input / output / residual may be channel slices of larger tensors, which
 * replaces torch.cat.  y = act(conv(pad(upsample(x))) + bias) * out_scale (+ residual).
 * ------------------------------------------------------------------------------------------ */
#define B200_ACT_NONE 0
#define B200_ACT_RELU 1
#define B200_ACT_LEAKY02 2
#define B200_ACT_SIGMOID 3
#define B200_ACT_TANH 4
#define B200_PAD_ZEROS 0
#define B200_PAD_REFLECT 1
#define B200_UP_NEAREST 0
#define B200_UP_BILINEAR_AC 1
typedef struct B200ConvDesc {
  int32_t N, Cin, H, W;            /* input extent (before the optional nearest upsample)            */
  int32_t in_c_total, in_c_off;    /* input = channels [in_c_off, in_c_off+Cin) of an in_c_total tensor */
  int32_t Cout, KH, KW, stride, pad_h, pad_w;
  int32_t pad_mode;                /* B200_PAD_*  (nn.Conv2d padding / nn.ReflectionPad2d)            */
  int32_t upsample;                /* 1, or 2 = nn.Upsample(scale_factor=2, mode='nearest') first     */
  int32_t out_c_total, out_c_off;
  int32_t act;                     /* B200_ACT_*                                                      */
  float out_scale;
  int32_t res_c_total, res_c_off;  /* residual tensor slice (same spatial size as the output)         */
  int32_t upsample_mode;           /* with upsample == 2: B200_UP_NEAREST or B200_UP_BILINEAR_AC
                                      (nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True),
                                      network_filter.py:22 — b200_conv2d_tma_chain only)               */
} B200ConvDesc;
int b200_conv2d(const B200ConvDesc* d, const float* x, const float* w, const float* bias,
                const float* residual, float* y, void* stream);
/* Tensor-core (wgmma, fp16 operands / fp32 accumulate) variant of b200_conv2d for the layers the reference
 * itself runs with 10-bit-mantissa operands (RAFT under fp16 autocast, core/raft.py:131; stage-2 cuDNN
 * convolutions with TF32 allowed).  Same descriptor semantics as b200_conv2d; stride 1 or 2.  The input slice is
 * first repacked to fp16 with padding / upsampling / stride phases materialised (workspace of
 * b200_conv_tma_workspace_bytes(d) bytes), then every filter tap is a tiled TMA box load feeding wgmma directly.
 * Weights are first packed into tap-major swizzled fp16 images:
 *   bytes = b200_conv_tma_weight_image_bytes(d);  b200_conv_tma_weight_images(d, w, images, stream);
 * then b200_conv2d_tma_chain takes `images` in place of w.
 *
 * b200_conv2d_tma_chain(d, x, NULL, images, bias, residual, y, NULL, NULL, 0, ws, ws_bytes, stream) is the plain
 * convolution.  The chained form skips the fp16 NHWC repack of a convolution's input when its producers wrote it directly:
 *   in_packed  (or NULL): the packed input of `d` — b200_conv_tma_workspace_bytes(d) bytes, 256-byte aligned, zeroed once
 *              by the caller (halo and padded channels stay zero), interior written by the producers; x and the
 *              workspace are then ignored
 *   out_packed (or NULL) + next + next_c_off: ALSO write act(conv) as fp16 into the packed input of the consumer
 *              convolution `next` at its input channel next_c_off (several producers may fill one consumer: concat);
 *              y may then be NULL (no fp32 NCHW output at all); the fp16 store saturates at +-65504 like the repack
 * Filters wider than 129 taps at stride 1 (258 at stride 2) are refused: the size functions return -1 for them.
 * `next` / `d` with a packed input must satisfy b200_conv_tma_chainable: stride 1, no upsampling, zero or reflection
 * padding (a reflection halo is mirrored from the interior by the consumer call), whole input tensor (no channel slice),
 * Cin * KW > 64. */
int64_t b200_conv_tma_workspace_bytes(const B200ConvDesc* d);
int64_t b200_conv_tma_weight_image_bytes(const B200ConvDesc* d);
int b200_conv_tma_weight_images(const B200ConvDesc* d, const float* w, void* images, void* stream);
int b200_conv_tma_chainable(const B200ConvDesc* next);
int b200_conv2d_tma_chain(const B200ConvDesc* d, const float* x, void* in_packed, const void* w_images,
                          const float* bias, const float* residual, float* y, void* out_packed,
                          const B200ConvDesc* next, int32_t next_c_off, void* workspace,
                          int64_t workspace_bytes, void* stream);
/* Packs an fp32 NCHW tensor x [next->N][C][next->H][next->W] as fp16 (saturating, like the repack) into the packed
 * input of the chainable consumer `next`, at its input channels [next_c_off, next_c_off + C): another producer of a
 * concatenated input, for a tensor no convolution writes (the ConvLSTM's previous hidden state).  Other channels of
 * out_packed are left as they are.  Refused unless C and next_c_off are multiples of 8 and the slice lies inside
 * next->Cin. */
int b200_conv_tma_pack_chain(const B200ConvDesc* next, const float* x, int32_t C, void* out_packed,
                             int32_t next_c_off, void* stream);
/* ConvLSTM (network_local.py:18-53) on the tensor cores: the gate convolution `d` (the reference's Gates layer,
 * Cout = 4C with C % 8 == 0, stride 1, act none, out_scale 1, no residual or output slice) with the cell update in
 * its epilogue, so the 4C-channel gates tensor is never written:
 *   cell = sigmoid(remember) * prev_cell + sigmoid(in) * tanh(cell_gate),  hidden = sigmoid(out) * tanh(cell)
 * with the reference's gate order (chunk(4, 1): in, remember, out, cell) and each product and the sum rounded to
 * fp32 as torch rounds them; prev_cell == NULL is the zero state (cell = sigmoid(in) * tanh(cell_gate)).
 * hidden, cell (may be NULL), prev_cell: fp32 [N][C][OH][OW].  x / in_packed / workspace as in b200_conv2d_tma_chain;
 * with a previous state the input is [x | prev_hidden] (Cin = 2C), e.g. a packed input whose channels [C, 2C) were
 * filled by b200_conv_tma_pack_chain.  The weight images are gate-interleaved (32-column block b of an N tile holds
 * the four gates of hidden channels 8b .. 8b+7, see DESIGN §4b): build them with b200_convlstm_tma_weight_images
 * from the reference's Gates.weight unchanged ([4C][Cin][KH][KW]); they take b200_conv_tma_weight_image_bytes(d)
 * bytes.  bias is the reference's Gates.bias unchanged. */
int b200_convlstm_tma_weight_images(const B200ConvDesc* d, const float* w, void* images, void* stream);
int b200_convlstm_tma(const B200ConvDesc* d, const float* x, void* in_packed, const void* w_images,
                      const float* bias, const float* prev_cell, float* hidden, float* cell, void* workspace,
                      int64_t workspace_bytes, void* stream);
int b200_maxpool2(const float* x, float* y, int64_t planes, int32_t H, int32_t W, void* stream);
int b200_upsample_bilinear2(const float* x, float* y, int32_t N, int32_t C, int32_t H, int32_t W,
                            int32_t out_c_total, int32_t out_c_off, void* stream);
/* nn.InstanceNorm2d(affine=False) per (n,c) plane (+ReLU) and relu(a+b): the RAFT encoder's residual
 * blocks (src/models/stage_1/core/extractor.py:6-57,118-192) */
int b200_instance_norm(const float* x, float* y, int64_t planes, int64_t hw, float eps, int32_t relu,
                       void* stream);
int b200_add_relu(const float* a, const float* b, float* out, int64_t n, void* stream);
/* mode 0: out = a*b (r*h into a concat buffer); mode 1: out = (1-a)*b + a*c (GRU state update) */
int b200_gru_gate(const float* a, const float* b, const float* c, float* out, int64_t n_per_sample,
                  int64_t samples, int64_t out_sample_stride, int32_t mode, void* stream);
/* ConvLSTM cell on fp32 gates [N][4C][H][W] (pre-activation, chunk(4, 1) order) -> hidden, cell (may be NULL),
 * [N][C][H][W]; the same expressions as b200_convlstm_tma's epilogue.  prev_cell == NULL is the zero state;
 * b200_convlstm_zero_state(gates, ...) is b200_convlstm_cell(gates, NULL, ...). */
int b200_convlstm_cell(const float* gates, const float* prev_cell, float* hidden, float* cell, int32_t N,
                       int32_t C, int32_t H, int32_t W, void* stream);
int b200_convlstm_zero_state(const float* gates, float* hidden, float* cell, int32_t N, int32_t C,
                             int32_t H, int32_t W, void* stream);
/* RAFT.upsample_flow (core/raft.py:76-87): flow [N][2][H][W], mask [N][576][H][W] -> [N][2][8H][8W] */
int b200_convex_upsample(const float* flow, const float* mask, float* out, int32_t N, int32_t H,
                         int32_t W, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200_DEFLICKER_H */
