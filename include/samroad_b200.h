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

#define SAMROAD_ABI_VERSION 5

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

/* ---- threshold search: exact binary precision-recall curves ---------------------------------------- */

/* One accumulator stands for one torchmetrics BinaryPrecisionRecallCurve(thresholds=None,
 * ignore_index=-1) of SAMRoad (model.py:361-363), fed by test_step (model.py:602-617) and read by
 * on_test_end (model.py:619-634).  Each kept entry is stored as one 32-bit key on the device (4 bytes);
 * compute needs 4 more bytes per entry and 28 bytes per distinct score while it runs.  At most 2^31-1
 * entries per accumulator.  Calls on one handle are ordered on the stream they are given. */
typedef struct samroad_prc_ctx* samroad_prc_t;

int samroad_prc_create(int device, samroad_prc_t* out);
int samroad_prc_destroy(samroad_prc_t p);
/* Drops every entry (torchmetrics' reset()).  Asynchronous. */
int samroad_prc_reset(samroad_prc_t p, void* stream);
/* Appends n entries; asynchronous, no host synchronisation.  preds: device fp32, element i at
 * preds[i * pred_stride] (so mask_scores[..., c] of [B,P,P,2] is read in place with stride 2).
 * target: n contiguous SAMROAD_F32 values (label = int32(target), truncating as .to(torch.int32) does)
 * or SAMROAD_U8 bytes.  valid: NULL or n bytes, 0 = ignored (the reference's target -1).
 * An update with a kept prediction that is NaN or outside [0, 1] (torchmetrics would apply a sigmoid to
 * the whole batch instead) or a kept label other than 0 / 1 (torchmetrics raises) adds nothing; the next
 * samroad_prc_compute or samroad_prc_export_keys fails with code 3 and reports every refused update since
 * the last report (their number, the first in detail), and the handle stays usable. */
int samroad_prc_update(samroad_prc_t p, const float* preds, int64_t pred_stride, const void* target,
                       int target_dtype, const uint8_t* valid, int64_t n, void* stream);
/* Distributed evaluation (one accumulator per rank; the curve of the whole split needs every rank's
 * entries, as torchmetrics' sync on compute gathers them): export_keys synchronises, reports refused
 * updates like compute, writes the number of accepted entries to *n_keys and, when keys != NULL, copies
 * their packed 32-bit keys (any order) into keys (device or host, room for cap).  append_keys adds keys
 * exported by other accumulators (device memory, asynchronous); a key whose score is outside [0, 1]
 * refuses the call like a bad update. */
int samroad_prc_export_keys(samroad_prc_t p, uint32_t* keys, int64_t cap, int64_t* n_keys, void* stream);
int samroad_prc_append_keys(samroad_prc_t p, const uint32_t* keys, int64_t n, void* stream);
/* Sorts the entries and builds the curve (synchronises).  counts (host, 4): entries, positives,
 * distinct thresholds T, index of the best point.  best (host, 4): threshold, precision, recall and F1 at
 * the first maximum of F1 = 2*(P*R)/(P+R), a NaN F1 counting as larger than any number (torch.argmax).
 * Counts are exact integers; P, R and F1 are the float32 operations of the reference in its order. */
int samroad_prc_compute(samroad_prc_t p, int64_t* counts, float* best, void* stream);
/* The curve of the last successful compute in torchmetrics' layout, each pointer may be NULL (device or
 * host memory): thresholds [T] ascending, precision / recall [T+1] ending with the point (1, 0), and
 * the int64 true / false positive counts [T] at each threshold (score >= threshold).  Asynchronous. */
int samroad_prc_read_curve(samroad_prc_t p, float* thresholds, float* precision, float* recall,
                           int64_t* tps, int64_t* fps, void* stream);

/* ---- validation: losses, IoUs and F1 of validation_step / on_validation_epoch_end --------------------- */

/* One accumulator stands for the criteria and metrics of SAMRoad (model.py:349-359) as validation_step
 * (model.py:547-588) feeds them and on_validation_epoch_end (model.py:591-600) reads them: the epoch's
 * batch-size-weighted mean of the three step losses, and exact int64 confusion counts of the keypoint mask,
 * the road mask and the valid pair slots (prediction positive when score > 0.5).  O(1) device state.  Calls
 * on one handle are ordered on the stream they are given. */
typedef struct samroad_val_ctx* samroad_val_t;

#define SAMROAD_LOSS_BCE 0   /* BCEWithLogitsLoss() */
#define SAMROAD_LOSS_FOCAL 1 /* torchvision sigmoid_focal_loss(alpha=0.25, gamma=2, reduction='mean') */

int samroad_val_create(int device, samroad_val_t* out);
int samroad_val_destroy(samroad_val_t v);
/* Clears the epoch state (counts, loss sums) and any unreported refusal.  Asynchronous. */
int samroad_val_reset(samroad_val_t v, void* stream);
/* One validation step; asynchronous, no host synchronisation.  Device pointers:
 *   mask_logits, mask_scores  [B,P,P,2] float32 as samroad_encode_masks writes them (8-byte aligned);
 *   keypoint_mask, road_mask  [B,P,P] float32 targets, each exactly 0.0 or 1.0;
 *   topo_logits, topo_scores  [B*Ns*Np] float32; connected, valid [B*Ns*Np] bytes, 0 or 1;
 *   out                       [3] float32: the step's (mask_loss, topo_loss, loss).
 * mask_loss is the mean of the per-element loss (loss_kind) over both channels, topo_loss the mean of the
 * BCE over the valid slots (NaN without one), loss = mask_loss + topo_loss; the element terms are the
 * reference's float32 expressions, their sums fp64, each mean rounded to float32 once.  A step with a mask
 * target other than 0.0 / 1.0, a counted score that is NaN or outside [0, 1], or a connected / valid byte
 * other than 0 / 1 is refused as a whole: it adds nothing and writes NaN to out; the next samroad_val_read
 * fails with code 3 and reports every refused step since the last report (their number, the first in
 * detail: element index e < 2*B*P*P is mask entry e of [B,P,P,2], above it pair slot e - 2*B*P*P), and the
 * handle stays usable. */
int samroad_val_update(samroad_val_t v, const float* mask_logits, const float* mask_scores,
                       const float* keypoint_mask, const float* road_mask, const float* topo_logits,
                       const float* topo_scores, const uint8_t* connected, const uint8_t* valid, int B, int P,
                       int Ns, int Np, int loss_kind, float* out, void* stream);
/* Synchronises and reports refused steps (see update).  Host outputs:
 *   counts [11] int64: keypoint tp, fp, fn, tn; road tp, fp, fn, tn; topology tp, fp, fn (valid slots);
 *   means  [3] float32: epoch (mask_loss, topo_loss, loss) = f32(sum(step value * B) / sum(B)), NaN
 *          before the first accepted step;
 *   totals [2] int64: accepted steps, sum of their B. */
int samroad_val_read(samroad_val_t v, int64_t* counts, float* means, int64_t* totals, void* stream);

/* ---- training of the heads with a frozen encoder: SAMRoad.training_step (model.py:511-544) ---------------- */

/* One step of FREEZE_ENCODER training (naive map decoder + TopoNet; USE_SAM_DECODER is refused).  The
 * encoder runs as in samroad_encode_masks; the heads run in fp32 from the caller's parameters, given as a
 * table of (state_dict key, device fp32 pointer in the reference layout): every map_decoder.* and topo_net.*
 * parameter of the configuration.  Backward regenerates the dropout masks from (seed, layer, site, element). */
typedef struct SamRoadTrainArgs {
  int32_t B, N, Ns, Np;   /* tiles, points per tile, samples per tile, pairs per sample (1..32)          */
  int32_t loss_kind;      /* SAMROAD_LOSS_BCE or SAMROAD_LOSS_FOCAL (mask criterion)                      */
  float dropout_p;        /* TopoNet dropout: 0.1 in training mode, 0 in eval mode                        */
  uint64_t seed;          /* dropout seed                                                                 */
} SamRoadTrainArgs;

/* Bytes of the workspace one step needs: forward activations kept for backward plus backward scratch. */
int samroad_train_workspace_bytes(samroad_handle_t h, const SamRoadTrainArgs* args, size_t* bytes);
/* Forward of one step; asynchronous.  Device inputs as samroad_encode_masks / samroad_toponet take them, plus
 * connected [B,Ns,Np] bytes and keypoint_mask / road_mask [B,P,P] fp32 targets (any finite value).  Writes
 * losses[2] = (mask_loss, topo_loss) (device fp32; topo_loss is NaN without a valid slot, as in the
 * reference), keeps what backward needs in ws, and copies the image embeddings [B,256,P/16,P/16] when
 * image_embeddings != NULL. */
int samroad_train_forward(samroad_handle_t h, const SamRoadTrainArgs* args, const char* const* keys,
                          const float* const* params, int n_params, const void* rgb, int rgb_dtype,
                          const void* points, int pts_dtype, const void* pairs, int pairs_dtype,
                          const uint8_t* valid, const uint8_t* connected, const float* keypoint_mask,
                          const float* road_mask, void* ws, size_t ws_bytes, float* losses,
                          float* image_embeddings, void* stream);
/* Backward of the step whose forward filled ws (ws is not modified where forward wrote it, so backward may
 * run more than once); asynchronous.  g: device fp32 [2] = incoming gradients of (mask_loss, topo_loss).
 * Writes (overwrites) the gradient of every parameter of the table into grads[i] (device fp32, reference
 * layout).  Deterministic: no float atomics. */
int samroad_train_backward(samroad_handle_t h, const SamRoadTrainArgs* args, const char* const* keys,
                           const float* const* params, float* const* grads, int n_params, void* ws,
                           size_t ws_bytes, const float* g, void* stream);
/* Forward of one step of the heads on caller-supplied image embeddings (device fp32 [B,256,P/16,P/16], NCHW,
 * contiguous) in place of rgb: the encoder does not run; the embeddings are copied into ws and everything
 * downstream is samroad_train_forward's.  Same arguments and outputs otherwise. */
int samroad_train_forward_embeddings(samroad_handle_t h, const SamRoadTrainArgs* args, const char* const* keys,
                                     const float* const* params, int n_params, const float* image_embeddings,
                                     const void* points, int pts_dtype, const void* pairs, int pairs_dtype,
                                     const uint8_t* valid, const uint8_t* connected, const float* keypoint_mask,
                                     const float* road_mask, void* ws, size_t ws_bytes, float* losses,
                                     void* stream);
/* samroad_train_backward plus the gradient of the image embeddings, for a ws filled by either forward.
 * grads == NULL skips the weight gradients; grad_embeddings (device fp32 [B,256,P/16,P/16], NCHW, overwritten)
 * may be NULL, but not both.  The map decoder's and TopoNet's parts (through the bilinear sampler) are summed per
 * element in that order and scaled by g[0] / (2 B P^2) and g[1] / sum(valid) in fp32; a part whose incoming
 * gradient is exactly 0 adds nothing.  Deterministic: no float atomics. */
int samroad_train_backward_embeddings(samroad_handle_t h, const SamRoadTrainArgs* args, const char* const* keys,
                                      const float* const* params, float* const* grads, int n_params, void* ws,
                                      size_t ws_bytes, const float* g, float* grad_embeddings, void* stream);
/* Repacks one head tensor (map_decoder.* / topo_net.*) of finalized weights from DEVICE fp32 memory,
 * stream-ordered; the packed result equals what samroad_finalize_weights makes from the same values, bit for
 * bit.  Encoder tensors and the SAM mask decoder are refused. */
int samroad_update_tensor_device(samroad_handle_t h, const char* key, const float* dev_data,
                                 const int64_t* shape, int ndim, void* stream);
/* Test hook: keep[i] = 1 when element i of dropout site `site` (0 attention probabilities [rows,4,Np,Np],
 * 1 dropout1, 2 the dropout between ReLU and linear2, 3 dropout2, each [tokens,128]) of TopoNet layer `layer`
 * survives at rate 1 - p under `seed`, else 0. */
int samroad_debug_train_dropout_keep(float p, uint64_t seed, int layer, int site, int64_t n, uint8_t* keep,
                                     void* stream);

/* ---- training / evaluation batches on the device (sam_road_b200/dataset.py, DESIGN.md §13) ----
 * A labels object holds the scenes of one dataset: each scene's subdivided ground-truth graph as
 * GraphLabelGenerator.__init__ (dataset.py:71-125) builds it, precomputed on the host, and its uint8 RGB and
 * masks.  A batch runs GraphLabelGenerator.sample_patch (dataset.py:127-231) for B patches and collates them as
 * graph_collate_fn (dataset.py:287-302).  Not thread-safe; one batch at a time. */
typedef struct samroad_labels_ctx* samroad_labels_t;
typedef struct SamRoadLabelCfg {
  int32_t patch_size;            /* P                                                                      */
  int32_t image_size;            /* side of the (square) scenes                                            */
  int32_t sample_margin;         /* patch origins lie in [margin, image_size - P - margin]                 */
  int32_t topo_sample_num;       /* sources per patch (TOPO_SAMPLE_NUM) >= 1                               */
  int32_t max_neighbor_queries;  /* pairs per source (MAX_NEIGHBOR_QUERIES), 1..32                         */
  int32_t max_patch_points;      /* most non-excluded graph points any admissible P x P window holds       */
  double road_nms_radius;        /* ROAD_NMS_RADIUS > 0 (inclusive)                                        */
  double neighbor_radius;        /* NEIGHBOR_RADIUS > 0 (kNN strictly inside; BFS depth radius // 4 <= INT_MAX) */
} SamRoadLabelCfg;

int samroad_labels_create(int device, const SamRoadLabelCfg* cfg, samroad_labels_t* out);
int samroad_labels_destroy(samroad_labels_t L);
/* Copies one scene (host memory) to the device; *scene_index gets its index (upload order).  points [n,2]
 * float64 (x, y) of the subdivided graph; flags [n] bit 0 = excluded (near a crossover), bit 1 = never
 * suppressed by NMS (degree != 2); weights [n] sampling weights, each positive and finite; adj_start [n+1] /
 * adj CSR adjacency;
 * rgb [S,S,3], keypoint_mask / road_mask [S,S] uint8 with S = image_size. */
int samroad_labels_upload(samroad_labels_t L, const uint8_t* rgb, const uint8_t* keypoint_mask,
                          const uint8_t* road_mask, int32_t n_points, const double* points, const uint8_t* flags,
                          const float* weights, const int32_t* adj_start, const int32_t* adj,
                          int32_t* scene_index);
/* One batch of B patches on `stream`.  patches: device int32 [B,4] (scene, x0, y0, rot) or NULL to draw them
 * (training: uniform scene, origins in the margin range, rot 0..3).  Every other draw is Philox keyed by `seed`.
 * Outputs (device): rgb [B,P,P,3] float32 0..255, keypoint_mask / road_mask [B,P,P] float32 /255,
 * points [B,N,2] float32 (capacity B * max_patch_points * 2), pairs [B,S,Np,2] int32, connected / valid
 * [B,S,Np] bytes 0/1; *n_points = N (host), the largest point count of the batch.  Synchronises the stream once
 * to read the point counts. */
int samroad_labels_batch(samroad_labels_t L, int B, uint64_t seed, const int32_t* patches, float* rgb,
                         float* keypoint_mask, float* road_mask, float* points, int32_t* pairs,
                         uint8_t* connected, uint8_t* valid, int32_t* n_points, void* stream);
/* Test hook on the draw arrays of a batch (device or host memory): patches [B,4]; score_u [B,max_patch_points]
 * U[0,1) of the j-th candidate in ascending id; source_u [B,S] U[0,1); noise [B,max_patch_points,2] added to the
 * i-th point.  mode 0: the batch takes the caller-filled arrays instead of drawing them (seed unused).
 * mode 1: the batch draws as samroad_labels_batch(patches = NULL, seed) does and copies its draws out. */
int samroad_debug_labels_batch_draws(samroad_labels_t L, int B, int mode, uint64_t seed, int32_t* patches,
                                     double* score_u, double* source_u, double* noise, float* rgb,
                                     float* keypoint_mask, float* road_mask, float* points, int32_t* pairs,
                                     uint8_t* connected, uint8_t* valid, int32_t* n_points, void* stream);

/* ---- the TOPO graph metric (sam_road_b200/topo_metric.py, DESIGN.md §14) ----
 * A topo object holds one tile's two road graphs (0 ground truth, 1 proposal) as RoadGraph builds them
 * (cityscale_metrics/topo/graph.py) and scores (GT, proposal) pairs as TOPOWithPairs does: per pair the three
 * TOPOWalks, the candidate marble-hole edges and the two maximum matchings.  Capacities bound the device
 * workspaces; a run that exceeds one is refused with an error naming the pair, never truncated.  Not
 * thread-safe; one run at a time.  Synchronous (default stream). */
typedef struct samroad_topo_ctx* samroad_topo_t;
typedef struct SamRoadTopoCaps {
  int32_t max_marbles;      /* marbles (or holes) one walk may place                            */
  int32_t max_queue;        /* entries the FIFO of one walk may hold at once                     */
  int32_t max_covered;      /* directed edges one walk may sample (its edge_covered entries)     */
  int32_t max_candidates;   /* candidate marble-hole edges of one pair, per matching             */
  int32_t slots;            /* pairs in flight on the device at once                             */
} SamRoadTopoCaps;

int samroad_topo_create(int device, const SamRoadTopoCaps* caps, samroad_topo_t* out);
int samroad_topo_destroy(samroad_topo_t T);
/* Copies one graph (host memory) to the device, replacing the previous graph of that kind.  latlon [n,2] float64
 * (lat, lon) by node id; cos_lat [n] = math.cos(math.radians(lat)); link_start [n+1] / link: nodeLink, and
 * rlink_start [n+1] / rlink: nodeLinkReverse, each node's list in the reference's order.  Refuses a coordinate
 * that is not finite and an edge of length zero (naming it). */
int samroad_topo_upload_graph(samroad_topo_t T, int which, int32_t n_nodes, const double* latlon,
                              const double* cos_lat, const int32_t* link_start, const int32_t* link,
                              const int32_t* rlink_start, const int32_t* rlink);
/* Scores n_pairs pairs (host memory in and out).  pair_nodes [n,4] int32 (gpsn1, gpsn2, osmn1, osmn2): the
 * proposal edge and the GT edge of each pair; pair_dists [n,4] float64 (gpsd1, gpsd2, osmd1, osmd2).  r, step and
 * threshold as TOPOWithPairs takes them; cos40 = math.cos(math.radians(40)).  counts [n,6] int32 out: marbles,
 * holes, bidirectional holes, the maximum matching of marbles to bidirectional holes (precision), that of holes
 * to marbles (recall), and a status word that is 0 for every pair of a successful run. */
int samroad_topo_run(samroad_topo_t T, int32_t n_pairs, const int32_t* pair_nodes, const double* pair_dists,
                     double r, double step, double threshold, double cos40, int32_t* counts);

/* ---- the APLS graph metric (sam_road_b200/apls_metric.py, DESIGN.md §15) ----
 * An apls object holds one tile's two densified road graphs (0 ground truth, 1 proposal) as main.go's
 * GraphDensify builds them, with the directed integer arc weights int(GPSDistance(u, v) * 100.0) from the host.
 * It finds the snapping candidates of the control points and, per direction, the shortest paths between the
 * matched control points on both graphs and the pair score.  Capacities are per handle; a call past one is refused
 * with an error naming it, never truncated, and the handle stays usable.  Not thread-safe; one call at a time.
 * Synchronous (the handle's own non-blocking stream). */
#define SAMROAD_APLS_CANDIDATES 10
typedef struct samroad_apls_ctx* samroad_apls_t;
typedef struct SamRoadAplsCaps {
  int32_t max_nodes;            /* nodes of one graph                                            */
  int32_t max_arcs;             /* directed arcs of one graph (adjacency entries)                */
  int32_t max_control_points;   /* control points of one direction (also candidate queries)      */
} SamRoadAplsCaps;
typedef struct SamRoadAplsResult {
  int64_t pairs;                /* unordered pairs of control points                             */
  int64_t cc;                   /* penalty + scored                                              */
  int64_t penalty;              /* pairs with an unmatched control point: each adds 1            */
  int64_t skipped;              /* both matched, d1 <= min_distance_filter or unreachable        */
  int64_t scored;               /* both matched, d1 > min_distance_filter: adds min(|d1-d2|/d1, 1) */
  uint64_t sum_fixed[3];        /* the exact sum of all terms, a 192-bit integer with LSB 2^-128 */
  double sum;                   /* sum_fixed rounded once to the nearest double, ties to even    */
  int32_t n_sources_gt;         /* matched control points (rows of dist_gt)                      */
  int32_t n_sources_prop;       /* their distinct matches (rows of dist_prop)                    */
  int32_t terminals_gt;         /* nodes of the contracted graphs the shortest paths ran on      */
  int32_t terminals_prop;
} SamRoadAplsResult;

int samroad_apls_create(int device, const SamRoadAplsCaps* caps, samroad_apls_t* out);
int samroad_apls_destroy(samroad_apls_t A);
/* Copies one graph (host memory) to the handle, replacing the previous graph of that kind.  latlon [n,2] float64
 * (lat, lon) by node id; row_start [n+1] / col / weight: the directed arcs of each node with their weights in cm.
 * Any digraph is accepted: arcs need no reverse arc, and self-loops and repeated arcs are allowed (a repeated arc
 * counts with its lightest weight).  Refuses a coordinate that is not finite, a negative weight, and
 * weights that sum to 2^31 - 1 or more (a distance could then exceed int32). */
int samroad_apls_upload_graph(samroad_apls_t A, int which, int32_t n_nodes, const double* latlon,
                              const int32_t* row_start, const int32_t* col, const int32_t* weight);
/* For each query point (lat, lon), the SAMROAD_APLS_CANDIDATES nodes of graph `which` nearest to it by squared
 * distance to the node's [x - 1e-6, x + 1e-6] box in degree space, ties by ascending node id, nearest first;
 * -1 pads when the graph has fewer nodes.  out [n_queries, SAMROAD_APLS_CANDIDATES] int32. */
int samroad_apls_candidates(samroad_apls_t A, int which, int32_t n_queries, const double* query_latlon,
                            int32_t* out);
/* One direction of main.go's apls_one_way after the snapping: graph gt_role plays the ground truth.  cp_gt [n_cp]:
 * the control points, ascending node ids of graph gt_role; cp_match [n_cp]: the node of the other graph each is
 * matched to, or -1.  Shortest paths run from every matched control point to the others on graph gt_role, and
 * between their matches on the other graph; the pair score runs over every unordered pair.  dist_gt
 * [n_sources_gt, n_sources_gt] (matched control points in cp order) and dist_prop [n_sources_prop, n_sources_prop]
 * (distinct matches in order of first appearance) receive the distances in cm (-1: unreachable) when not NULL. */
int samroad_apls_one_way(samroad_apls_t A, int gt_role, int32_t n_cp, const int32_t* cp_gt, const int32_t* cp_match,
                         double min_distance_filter, SamRoadAplsResult* out, int32_t* dist_gt, int32_t* dist_prop);

/* ---- label masks of the datasets (sam_road_b200/label_masks.py, DESIGN.md §16) ----
 * cityscale/generate_labels.py and spacenet/generate_labels.py for T tiles of size x size pixels at once,
 * pixel-identical to OpenCV 4.x: cv2.circle(kp, p, keypoint_radius, 255, -1) at every keypoint and
 * cv2.line(road, p0, p1, 255, road_width) for every edge.  All pointers are device memory.  nodes_xy [n, 2] int32
 * (x, y) keypoint centres with node_off [T + 1] int64 (tile t owns rows node_off[t] .. node_off[t + 1] - 1);
 * edges_xyxy [m, 4] int32 (x0, y0, x1, y1) with edge_off [T + 1] int64 likewise.  Centres and end points may lie
 * outside the tile.  Writes uint8 [T, size, size] masks of 0 / 255, zeroed first.  Refuses, before any launch,
 * road_width outside [2, 32767] (width 1 is another OpenCV path), keypoint_radius outside [0, 32767], size < 1,
 * T < 0 and null pointers.  Stateless and asynchronous on `stream`. */
int samroad_label_masks(int T, int size, const int32_t* nodes_xy, const int64_t* node_off, const int32_t* edges_xyxy,
                        const int64_t* edge_off, int keypoint_radius, int road_width, uint8_t* keypoint_mask,
                        uint8_t* road_mask, void* stream);

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
/* out32[M,N] = A W^T + bias + resid + pos[m % pos_rows]   (bias/resid/pos may be NULL; resid, [M, ldo], may be
   out32; out32 and resid 16-byte aligned, ldo a multiple of 4 and >= N) */
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
/* The SAM mask decoder alone (USE_SAM_DECODER handles): the forward of samroad_encode_masks on caller-given
 * fp32 NCHW embeddings [B,256,s,s] with the handle's weights, then stream-ordered copies of four of its
 * intermediates (each may be NULL): queries [B,4,256] after norm_final_attn, keys [B,T,256] after the last
 * norm4, hyper [B,2,32] (hypernetworks of mask tokens 1, 2) and the low-res masks lowres [B,4s,4s,2].
 * Refused before any launch: a handle without the decoder, unfinalised weights, a NULL emb_nchw, B <= 0
 * and both mask outputs NULL. */
int samroad_op_sam_decoder(samroad_handle_t h, const float* emb_nchw, int B, float* queries, float* keys,
                           float* hyper, float* lowres, float* mask_scores, float* mask_logits, void* stream);

/* Caller buffers (device) for the intermediates of samroad_op_encoder_taps; every pointer may be NULL.
 * M = B * (P/16)^2 token rows, D = embed_dim; fp16 buffers are IEEE half. */
typedef struct SamroadEncoderTaps {
  float* tokens0;          /* [M, D] fp32: X after patch embed + pos_embed                                 */
  uint64_t block_mask;     /* bit i: copy X after block i                                                  */
  float* blocks;           /* [popcount(block_mask), M, D] fp32, the selected blocks in ascending order   */
  int32_t detail_block;    /* block whose operands go to the six buffers below; -1: none                  */
  void* ln1;               /* [M, D] fp16: norm1 output                                                    */
  void* qkv;               /* [M, 3D] fp16: qkv linear (LoRA merged), columns (q|k|v) x head x hd          */
  void* att;               /* [M, D] fp16: attention output, before proj                                   */
  float* x_attn;           /* [M, D] fp32: X after proj + residual                                         */
  void* ln2;               /* [M, D] fp16: norm2 output                                                    */
  void* h;                 /* [M, 4D] fp16: GELU(lin1)                                                     */
  void* n1;                /* [M, 256] fp16 NHWC: neck conv1 + LayerNorm2d                                 */
  void* feat16;            /* [M, 256] fp16 NHWC: neck output (the map decoder's A operand)                */
  void* d1;                /* [4M, 128] fp16: naive decoder stage 1, row (m * 4 + d), d = di * 2 + dj      */
  void* d2;                /* [16M, 64] fp16: naive decoder stage 2, row ((m * 4 + d1) * 4 + d2)           */
} SamroadEncoderTaps;

/* Test hook: exactly samroad_encode_masks, plus stream-ordered copies (no kernels) of the intermediates
 * `taps` selects, each made right after the launch that produces it.  taps == NULL is samroad_encode_masks.
 * d1 / d2 are written only when the naive decoder runs (a mask output is requested, no SAM decoder).
 * Refused before any launch: a NULL handle, a block_mask bit or a detail_block >= depth. */
int samroad_op_encoder_taps(samroad_handle_t h, const void* rgb, int rgb_dtype, int B,
                            const SamroadEncoderTaps* taps, float* mask_scores, float* mask_logits,
                            float* image_embeddings, void* stream);

/* Test hook: bit 0 routes samroad_op_attention / the encoder through the fp32 SIMT attention
 * kernel (the independent on-device checker of the tensor-core kernel).  Not for production use. */
void samroad_debug_force_simt_attention(int on);
/* Test hook: the kernel samroad_op_attention runs for grid s, window win and head_dim, as it would be chosen
 * now (no launch, no device needed): 0 the one-CTA-per-window kernel, 1 the streamed kernel, 2 the global
 * wgmma kernel, 3 the SIMT kernel (forced by samroad_debug_force_simt_attention).  *q_stages and *kv_stages
 * (each may be NULL) get the global kernel's Q and K/V ring depths, 0 on the other paths.  Returns -1 (see
 * samroad_last_error) for a shape or head_dim samroad_op_attention refuses. */
int samroad_debug_attention_path(int s, int win, int head_dim, int* q_stages, int* kv_stages);
/* Test hook (bit mask): bit 4 (16) makes the encoder's LayerNorms walk the token rows ascending
 * (by default those of even blocks walk them descending).  Other bits are ignored. */
void samroad_debug_disable_2cta_gemm(int off);

#ifdef __cplusplus
}
#endif
#endif /* SAMROAD_B200_H_ */
