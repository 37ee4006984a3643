/* samroad_b200.h -- C ABI of libsamroad_b200.so
 *
 * H100-native (sm_90a) implementation of the tiled-inference hot path of htcr/sam_road.
 * Every entry point replaces one piece of the reference's Python interface (file:line cited per
 * function, relative to the reference repository root).  The reference has no FFI of its own (it is
 * pure PyTorch, SURVEY.md §2.2); the binding a maintainer adds is the ctypes stub shown in
 * INTEGRATION.md, which is also what sam_road_b200/_lib.py implements.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary.
 *   - every function returns 0 on success; on failure a non-zero code is returned and
 *     samroad_last_error() (thread-local) describes the problem.  Nothing throws or aborts.
 *   - device pointers are caller-owned (e.g. torch tensors' data_ptr()); the handle owns only the
 *     packed weights and its activation workspace.
 *   - calls are asynchronous and ordered on the given cudaStream_t (passed as void*); one handle
 *     per device, not re-entrant on the same handle.  Multi-GPU = one process per GPU.
 *   - there is no CPU fallback: without a CUDA device every compute call fails.
 */
#ifndef SAMROAD_B200_H_
#define SAMROAD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SAMROAD_ABI_VERSION 4

typedef struct samroad_ctx* samroad_handle_t;

/* dtype codes for polymorphic inputs */
enum { SAMROAD_F32 = 0, SAMROAD_I64 = 1, SAMROAD_I32 = 2, SAMROAD_U8 = 3, SAMROAD_F64 = 4 };

/* TOPONET_VERSION (model.py:84,111-116,135).  'no_tgt_features' behaves as 'normal' in the
 * reference because the following if/else overwrites it (model.py:111-116). */
enum { SAMROAD_TOPO_NORMAL = 0, SAMROAD_TOPO_NO_OFFSET = 1, SAMROAD_TOPO_NO_TRANSFORMER = 2 };

/* Model hyper-parameters: what SAMRoad.__init__ derives from the YAML config (model.py:193-300). */
typedef struct SamRoadCfg {
  int32_t patch_size;             /* PATCH_SIZE: tile side in pixels, multiple of 16            */
  int32_t embed_dim;              /* 768 (vit_b) / 1024 (vit_l) / 1280 (vit_h)  model.py:198-218 */
  int32_t depth;                  /* 12 / 24 / 32                                               */
  int32_t num_heads;              /* 12 / 16 / 16                                               */
  int32_t window_size;            /* 14 (model.py:256)                                          */
  int32_t global_attn_indexes[4]; /* model.py:203,210,217                                       */
  int32_t use_sam_decoder;        /* USE_SAM_DECODER (model.py:260)                             */
  int32_t toponet_version;        /* SAMROAD_TOPO_*                                             */
  int32_t lora_rank;              /* 0 = no LoRA; else LORA_RANK (model.py:304-347)             */
} SamRoadCfg;

/* ---- lifetime ------------------------------------------------------------------------------ */

/* Replaces SAMRoad.__init__ + .to(device) (model.py:193-300, inferencer.py:247-254). */
int samroad_create(const SamRoadCfg* cfg, int device, samroad_handle_t* out);
int samroad_destroy(samroad_handle_t h);

/* Replaces load_state_dict (inferencer.py:250-252): hand over one fp32 tensor of the reference's
 * state_dict by its key (SURVEY.md §8b lists the key set) from HOST memory.  Unknown keys are an
 * error.  After all tensors are loaded call samroad_finalize_weights(), which packs them to the
 * device formats (fp16 K-major GEMM operands, LoRA merged into qkv, ConvTranspose re-ordered as
 * GEMM) and reports any missing key. */
int samroad_load_tensor(samroad_handle_t h, const char* key, const float* host_data,
                        const int64_t* shape, int ndim);
int samroad_finalize_weights(samroad_handle_t h);

/* ---- the hot path --------------------------------------------------------------------------- */

/* SAMRoad.infer_masks_and_img_features (model.py:459-495) and the mask half of forward()
 * (model.py:414-446).  rgb: device [B,P,P,3], SAMROAD_F32 (0..255) or SAMROAD_U8.
 * Outputs (device, fp32): mask_scores [B,P,P,2] (may be NULL), mask_logits [B,P,P,2] (may be NULL),
 * image_embeddings [B,256,P/16,P/16]. */
int samroad_encode_masks(samroad_handle_t h, const void* rgb, int rgb_dtype, int B,
                         float* mask_scores, float* mask_logits, float* image_embeddings,
                         void* stream);

/* The same for tiles that are windows of a uint8 RGB scene [H,W,3] already on the device: replaces
 * crop_img_patch / get_batch_img_patches + the per-batch float32 upload (inferencer.py:43-58,87-96).
 * tile_xy: device int32 [B,2] tile origins (x0,y0); the tile is scene[y0:y0+P, x0:x0+P, :]. */
int samroad_encode_masks_scene(samroad_handle_t h, const uint8_t* scene, int H, int W,
                               const int32_t* tile_xy, int B, float* mask_scores, float* mask_logits,
                               float* image_embeddings, void* stream);

/* SAMRoad.infer_toponet (model.py:498-508) = BilinearSampler (model.py:34-58) + TopoNet.forward
 * (model.py:88-148).  image_embeddings: device fp32 [B,256,s,s]; points [B,N,2] (x,y) pixels,
 * SAMROAD_F32 / I64 / I32; pairs [B,Ns,Np,2] indices into N, SAMROAD_I64 / I32; valid [B,Ns,Np]
 * bytes (0/1), Np = MAX_NEIGHBOR_QUERIES in 1..32.  Outputs fp32 [B,Ns,Np] (either may be NULL).
 * Slots masked by `valid` report output_proj.bias, mirroring torch's eval fast path (SURVEY.md §8a P4). */
int samroad_toponet(samroad_handle_t h, const float* image_embeddings, const void* points,
                    int pts_dtype, const void* pairs, int pairs_dtype, const uint8_t* valid, int B,
                    int N, int Ns, int Np, float* topo_logits, float* topo_scores, void* stream);

/* Mask fusion of inferencer.py:79-110: scores device fp32 [n_tiles,P,P,2] in tile-list order,
 * tile origins (device int32) -> uint8 [H,W] keypoint and road masks (device). */
int samroad_fuse_masks(const float* scores, int n_tiles, int P, const int32_t* tile_x0,
                       const int32_t* tile_y0, int H, int W, uint8_t* keypoint_u8,
                       uint8_t* road_u8, void* stream);

/* Same as samroad_encode_masks but with HOST buffers (pinned or pageable): uploads the uint8 / fp32
 * tiles, runs the path, downloads the results and synchronises.  This is the end-to-end call the
 * benchmark's `e2e` figure times.  Any output pointer may be NULL. */
int samroad_encode_masks_host(samroad_handle_t h, const void* rgb_host, int rgb_dtype, int B,
                              float* mask_scores_host, float* image_embeddings_host);

/* One whole batch with HOST buffers: uploads tiles (and TopoNet inputs), runs encoder + mask head
 * (+ TopoNet when points_host != NULL), downloads mask scores [B,P,P,2], image embeddings
 * [B,256,s,s] and topology scores [B,Ns,Np], then synchronises.  Any output may be NULL.  This is
 * the call the benchmark's `e2e` figure times (what inferencer.py:87-104,195-206 does per batch). */
int samroad_infer_batch_host(samroad_handle_t h, const void* rgb_host, int rgb_dtype, int B,
                             const void* points_host, int pts_dtype, const void* pairs_host,
                             int pairs_dtype, const uint8_t* valid_host, int N, int Ns, int Np,
                             float* mask_scores_host, float* image_embeddings_host,
                             float* topo_scores_host);

/* ---- scene graph: the host code between and after the two model passes, on the device ---------- */

typedef struct samroad_graph_ctx* samroad_graph_t;

/* Scratch owner for the three calls below (one per device / scene driver). */
int samroad_graph_create(int device, samroad_graph_t* out);
int samroad_graph_destroy(samroad_graph_t g);

/* Optional host callback standing for `numpy.argsort(keys)` (ascending, NumPy's default kind).
 * keys: n values of key_dtype (SAMROAD_U8 mask scores, SAMROAD_F64 priorities); order_out: n int64.
 * Returns 0 on success.  graph_utils.nms_points visits candidates in `argsort(scores)[::-1]` order
 * (graph_utils.py:574); the order of EQUAL scores is an implementation detail of NumPy's unstable
 * sort (it differs between CPUs), so a caller that needs the reference's exact keypoints on this host
 * passes NumPy's permutation in; with NULL the device sorts as argsort(kind='stable')[::-1] would.
 * The callback may be invoked from up to three library threads at once (the three sorts of one call
 * are independent) and must be thread-safe. */
typedef int (*samroad_argsort_fn)(const void* keys, int key_dtype, int64_t n, int64_t* order_out,
                                  void* user);

/* graph_extraction.extract_graph_points (graph_extraction.py:130-139) including
 * get_points_and_scores_from_mask (graph_extraction.py:24-28) and the three graph_utils.nms_points
 * passes (graph_utils.py:572-591: greedy radius NMS in descending score order, inclusive radius,
 * scores > 1.0 never suppressed).  keypoint_mask / road_mask: device uint8 [H,W] (the fused masks of
 * inferencer.py:106-110); thresholds are config.*_THRESHOLD * 255 (compared as `mask > thr`).
 * Output: device int64 [n,2] (x,y) in the reference's order, *n_points on the host.  stats (host,
 * optional, 16 ints): candidates of the two masks, survivors of passes 1-2, NMS rounds of the three
 * passes, n; then microseconds of host wall clock: candidates, ordering of the three passes, NMS of the
 * three passes, total.  Synchronises the stream. */
int samroad_extract_graph_points(samroad_graph_t g, const uint8_t* keypoint_mask,
                                 const uint8_t* road_mask, int H, int W, double itsc_thr255,
                                 double road_thr255, double itsc_radius, double road_radius,
                                 samroad_argsort_fn argsort, void* user, int64_t* points_xy, int cap,
                                 int* n_points, int32_t* stats, void* stream);

/* Pair-query construction of inferencer.py:126-197 for every tile of the scene: the box query
 * (rtree.intersection, inclusive bounds, ascending point index) and the per-tile kNN
 * (KDTree.query(k=MAX_NEIGHBOR_QUERIES+1, distance_upper_bound=NEIGHBOR_RADIUS) minus self: strictly
 * closer than the radius, ascending distance, equal distances in ascending index) for
 * max_nbr = MAX_NEIGHBOR_QUERIES in 1..32.  points_xy: device int64 [N,2]; tile_xy_host: host int32
 * [n_tiles,2] tile origins (x0,y0) in tile-list order.  Writes the number of points of every tile to
 * tile_counts_host (the caller pads each batch to its own maximum, inferencer.py:179-185).  The plan
 * serves fill / aggregate calls with any K <= max_nbr.  Synchronises the stream. */
int samroad_pair_queries_plan_k(samroad_graph_t g, const int64_t* points_xy, int N,
                                const int32_t* tile_xy_host, int n_tiles, int P, double radius,
                                int max_nbr, int32_t* tile_counts_host, void* stream);
/* samroad_pair_queries_plan_k with max_nbr = 16. */
int samroad_pair_queries_plan(samroad_graph_t g, const int64_t* points_xy, int N,
                              const int32_t* tile_xy_host, int n_tiles, int P, double radius,
                              int32_t* tile_counts_host, void* stream);
/* Padded batch tensors for tiles [tile_begin, tile_begin+B): points int32 [B,nmax,2] relative to the
 * tile origin, pairs int32 [B,nmax,K,2], valid bytes [B,nmax,K] (device) -- the inputs of
 * samroad_toponet (inferencer.py:164-197).  K may not exceed the planned max_nbr.  Asynchronous. */
int samroad_pair_queries_fill(samroad_graph_t g, int tile_begin, int B, int nmax, int K,
                              int32_t* points, int32_t* pairs, uint8_t* valid, void* stream);

/* Edge aggregation of inferencer.py:206-230 over the planned tiles: topo_scores is one device fp32
 * buffer, tile t's scores [nmax_of_its_batch, K] start at element tile_score_offset_host[t] (negative:
 * the tile's batch was skipped, inferencer.py:188-189).  Per directed (src,tgt) the scores are added in
 * float32 in (tile, sample, pair) order, averaged and compared with `> threshold`; surviving edges are
 * written in first-occurrence order as int64 [n,2] global point indices.  *bad_score != 0 when a score
 * fell outside [0,1] (the reference asserts).  K may not exceed the planned max_nbr.  Synchronises the
 * stream. */
int samroad_aggregate_edges(samroad_graph_t g, const float* topo_scores,
                            const int64_t* tile_score_offset_host, int K, float threshold,
                            int64_t* edges, int cap, int* n_edges, int* bad_score, void* stream);

/* The pipelined form of samroad_infer_batch_host: queue one batch on staging slot 0 or 1 and return;
 * samroad_infer_batch_host_wait(h, slot) blocks until that batch's results are in host memory.  With
 * the two slots alternating, the downloads of batch i overlap the upload and the compute of batch
 * i+1 (what a scene driver streaming batches does).  Host buffers must stay valid (and should be
 * page-locked) until the wait returns. */
int samroad_infer_batch_host_async(samroad_handle_t h, int slot, const void* rgb_host, int rgb_dtype,
                                   int B, const void* points_host, int pts_dtype,
                                   const void* pairs_host, int pairs_dtype, const uint8_t* valid_host,
                                   int N, int Ns, int Np, float* mask_scores_host,
                                   float* image_embeddings_host, float* topo_scores_host);
int samroad_infer_batch_host_wait(samroad_handle_t h, int slot);

/* Stream memory operations on a 32-bit flag word in device (or peer-mapped) memory, executed by the stream
 * front end without a kernel: an ordered write of `value`, and a wait until *addr >= value.  The exchange step
 * between ranks (sam_road_b200/exchange.py; no reference counterpart, the reference is single-GPU) builds its
 * barrier from them so that no SM spins beside the persistent compute kernels. */
int samroad_stream_write_value32(void* addr, uint32_t value, void* stream);
int samroad_stream_wait_value32(void* addr, uint32_t value, void* stream);

/* Per-kernel-class CUDA-event timing on the launching stream (bench.py's roofline numbers).
 * samroad_timing_enable(h, 1) clears and starts recording; samroad_timing_read() synchronises and
 * writes a JSON object {"<class>": {"launches","ms","flops","bytes"}, ...} into buf. */
int samroad_timing_enable(samroad_handle_t h, int on);
int samroad_timing_read(samroad_handle_t h, char* buf, size_t cap);

/* Activation workspace the handle needs for a batch of B tiles (bytes). */
size_t samroad_workspace_bytes(samroad_handle_t h, int B);

/* Number of kernels launched by this library since the last call with reset != 0. */
uint64_t samroad_launch_count(int reset);

const char* samroad_last_error(void);
int samroad_abi_version(void);

/* ---- op-level entry points (unit tests and composition; all pointers device, fp16 = IEEE half) ---- */

/* out16[M,N] = act(A[M,K] W[N,K]^T + bias)      act: 0 none, 1 GELU(erf), 2 ReLU; others are rejected */
int samroad_op_gemm_f16(const void* A, int lda, const void* W, int ldw, int M, int N, int K,
                        const float* bias, int act, void* out16, int ldo, void* stream);
/* out32[M,N] = A W^T + bias + resid + pos[m % pos_rows]   (bias/resid/pos may be NULL) */
int samroad_op_gemm_f32(const void* A, int lda, const void* W, int ldw, int M, int N, int K,
                        const float* bias, const float* resid, const float* pos, int pos_rows,
                        float* out32, int ldo, void* stream);
/* grouped LayerNorm epilogue, see gemm_tc.cuh EpiLN (act as for samroad_op_gemm_f16) */
int samroad_op_gemm_ln(const void* A, int lda, const void* W, int ldw, int M, int N, int K,
                       const float* bias, const float* resid, const float* gamma,
                       const float* beta, float eps, int group, int act, void* out16, float* out32,
                       float* out_nchw, int tokens, int ldo, void* stream);
/* independent SIMT checker GEMM: out32 = A W^T */
int samroad_op_gemm_ref(const void* A, int lda, const void* W, int ldw, int M, int N, int K,
                        float* out32, int ldo, void* stream);
int samroad_op_layernorm(const float* x, const float* gamma, const float* beta, float eps, int M,
                         int D, void* out16, void* stream);
int samroad_op_attention(const void* qkv16, const float* qkv_bias, const float* rel_h,
                         const float* rel_w, int B, int s, int win, int heads, int head_dim,
                         void* out16, void* stream);

/* Test hook: bit 0 routes samroad_op_attention / the encoder through the fp32 SIMT attention
 * kernel (the independent on-device checker of the tensor-core kernel).  Not for production use. */
void samroad_debug_force_simt_attention(int on);
/* Test hook (bit mask): bit 4 (16) makes the encoder's LayerNorms walk the token rows ascending
 * (by default those of even blocks walk them descending).  Other bits are ignored. */
void samroad_debug_disable_2cta_gemm(int off);

#ifdef __cplusplus
}
#endif
#endif /* SAMROAD_B200_H_ */
