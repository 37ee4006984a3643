// sam_road_b200 :: handle, weight packing and the forward orchestration behind the C ABI.
//
// Reference call stack reproduced (SURVEY.md §3.1): SAMRoad.infer_masks_and_img_features
// (model.py:459-495) -> ImageEncoderViT.forward (image_encoder.py:106-116) -> map_decoder
// (model.py:284-295,490-491); SAMRoad.infer_toponet (model.py:498-508) -> BilinearSampler
// (model.py:34-58) -> TopoNet.forward (model.py:88-148).
#include "../../include/samroad_b200.h"

#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "common.cuh"
#include "ops.h"

using namespace srb;

namespace {

struct HostTensor {
  std::vector<int64_t> shape;
  std::vector<float> data;
  int64_t numel() const {
    int64_t n = 1;
    for (auto d : shape) n *= d;
    return n;
  }
};

struct BlockW {
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  __half* qkv_w;  float* qkv_b;
  __half* proj_w; float* proj_b;
  float *rel_h, *rel_w;
  __half* lin1_w; float* lin1_b;
  __half* lin2_w; float* lin2_b;
  int win;   // attention window (14) or s for global blocks
};

// ---- one region of the packed weights (packed_regions) ----
// Values samroad_finalize_weights computes on the host from a region's sources before it packs them.
enum HostStep {
  HS_NONE,
  HS_LORA_QKV,   // sources qkv, A_q, B_q, A_v, B_v: the qkv weight with the LoRA products merged in
  HS_DENSE_PE,   // source: the Gaussian matrix of the prompt encoder; the dense positional encoding [s, s, 256]
};

struct Source {
  std::string key;              // state_dict key
  std::vector<int64_t> shape;   // its required shape
  int64_t at;                   // element offset of its values in the region
};

struct Region {
  int pack;                  // Pack
  int64_t n;                 // elements
  int cin, cout;             // PK_CONVT: channels; PK_TILE4: bias length in cout
  HostStep host;
  bool refresh;              // samroad_update_tensor_device may rewrite it
  std::vector<Source> src;
};

// Where samroad_update_tensor_device packs one key: a refreshable region, its storage and the key's source in it.
struct RefreshTarget {
  Region r;
  void* dst;
  Source src;
};

}  // namespace

// Per-kernel-class CUDA-event timing (bench.py roofline): events are recorded on the launching
// stream around every launch while enabled; totals are read back with samroad_timing_read().
struct KernelTimer {
  struct Rec { int tag; double flops; double bytes; cudaEvent_t a, b; };
  bool on = false;
  std::vector<Rec> recs;
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  cudaEvent_t get() {
    if (used == pool.size()) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      pool.push_back(e);
    }
    return pool[used++];
  }
  void begin(int tag, double flops, double bytes, cudaStream_t st) {
    if (!on) return;
    Rec r{tag, flops, bytes, get(), get()};
    cudaEventRecord(r.a, st);
    recs.push_back(r);
  }
  void end(cudaStream_t st) {
    if (!on) return;
    cudaEventRecord(recs.back().b, st);
  }
  void reset() { recs.clear(); used = 0; }
};

enum KTag {
  KT_PATCH_IM2COL = 0, KT_GEMM_PATCH, KT_LAYERNORM, KT_GEMM_QKV, KT_ATTN_WINDOW, KT_ATTN_GLOBAL,
  KT_GEMM_PROJ, KT_GEMM_LIN1, KT_GEMM_LIN2, KT_NECK, KT_DECODER, KT_TOPO_SAMPLE, KT_TOPO_GEMM,
  KT_TOPO_PAIR, KT_TOPO_ATTN, KT_TOPO_OUT, KT_COUNT
};
static const char* kTagNames[KT_COUNT] = {
  "patch_im2col", "gemm_patch_embed", "layernorm", "gemm_qkv", "attention_window",
  "attention_global", "gemm_proj", "gemm_mlp_lin1", "gemm_mlp_lin2", "neck", "map_decoder",
  "topo_sample", "topo_gemm", "topo_pair_features", "topo_attention", "topo_output"};

struct samroad_ctx {
  SamRoadCfg cfg;
  KernelTimer timer;
  int device = 0;
  int s = 0, T = 0, D = 0, hd = 0;
  bool finalized = false;
  std::map<std::string, HostTensor> staged;

  // device weight arena
  std::vector<DeviceBuffer> weight_allocs;
  // the refreshable regions by state_dict key, filled by samroad_finalize_weights from packed_regions
  std::map<std::string, std::vector<RefreshTarget>> refresh_targets;

  // encoder
  __half* pe_w = nullptr; float* pe_b = nullptr; float* pos = nullptr;
  std::vector<BlockW> blocks;
  __half* neck0_w = nullptr; float *neck1_g = nullptr, *neck1_b = nullptr;
  __half* neck2_w = nullptr; float *neck3_g = nullptr, *neck3_b = nullptr;
  // naive decoder
  __half* dec1_w = nullptr; float* dec1_b = nullptr; float *dec_ln_g = nullptr, *dec_ln_b = nullptr;
  __half* dec2_w = nullptr; float* dec2_b = nullptr;
  __half* dec3_w = nullptr; float* dec3_b = nullptr;
  float* dec4_w = nullptr; float* dec4_b = nullptr;
  // SAM mask-decoder path (USE_SAM_DECODER)
  SamDecoderWeights sam{};
  DeviceBuffer sam_ws;
  // toponet
  __half* tp_feat_w = nullptr; float* tp_feat_b = nullptr;
  __half* tp_st_w = nullptr; float* tp_off_w = nullptr; float* tp_pair_b = nullptr;
  TopoLayerParams tp_layers[3];
  // fp16 layer weights [18*128, 128]: per layer Wq, Wk, Wv, Wo, W1, W2 as [128, 128] blocks, so that
  // in_proj_weight (Wq|Wk|Wv), out_proj, linear1 and linear2 are each one contiguous [N, 128] operand
  __half* tp_chunks = nullptr;
  float* tp_out_w = nullptr; float* tp_out_b = nullptr;

  // activation workspace (grown on demand); TopoNet has its own so that the encoder of the next scene
  // (another stream) can run while the TopoNet pass of the previous one is still in flight
  DeviceBuffer ws;
  DeviceBuffer topo_ws;
  // staging for the host-buffer entry points: two slots so that step i's downloads overlap step
  // i+1's upload and compute (samroad_infer_batch_host_async / _wait)
  struct HostSlot {
    DeviceBuffer in;                                      // tiles + TopoNet inputs + topology scores
    DeviceBuffer scores;
    DeviceBuffer emb;
    cudaEvent_t ev_h2d = nullptr, ev_emb = nullptr, ev_scores = nullptr, ev_compute = nullptr, ev_done = nullptr;
  };
  HostSlot slots[2];
  cudaStream_t s_h2d = nullptr, s_compute = nullptr, s_copy = nullptr;   // upload / compute / download
  cudaEvent_t ev_emb_hook = nullptr;                     // recorded once the embeddings are final (after the neck)
  const SamroadEncoderTaps* taps = nullptr;              // set for the duration of samroad_op_encoder_taps
};

namespace {

constexpr float kPixelMean[3] = {123.675f, 116.28f, 103.53f};   // model.py:229
constexpr float kPixelStd[3] = {58.395f, 57.12f, 57.375f};      // model.py:230

// test hook (bit 4 of samroad_debug_disable_2cta_gemm): every encoder LayerNorm walks its rows ascending
bool g_ln_ascending = false;

std::string fmt_key(const char* fmt, int i) {
  char buf[256];
  snprintf(buf, sizeof(buf), fmt, i);
  return buf;
}

bool is_global_block(const SamRoadCfg& c, int i) {
  for (int k = 0; k < 4; ++k)
    if (c.global_attn_indexes[k] == i) return true;
  return false;
}

// Grows a workspace or staging buffer to `need` bytes.  The handle's three streams may still read the old
// block, so the device is synchronised before it is replaced.
int grow(DeviceBuffer& b, size_t need, const char* what) {
  if (need <= b.capacity()) return 0;
  if (b.get()) SRB_CUDA_OK(cudaDeviceSynchronize());
  return b.reserve(need, what);
}

// ---- packed weights ------------------------------------------------------------------------------------------
// Every state_dict tensor reaches the device through one list (packed_regions) and one kernel (pack_kernel):
// samroad_finalize_weights walks the list and packs the staged host values, and indexes the refreshable regions by
// key; samroad_update_tensor_device packs one head tensor from device memory through that index.  So the two write
// the same bytes, and a refresh costs one map lookup.

// How a source is laid out in its region: dst[i] = src[j(i)], fp16 rounded to nearest even or fp32.
enum Pack {
  PK_F32,        // fp32 copy
  PK_F16,        // fp16 copy: an nn.Linear weight [out, in] is already the K-major [N, K] operand
  PK_PATCH,      // patch embed [D,3,16,16] -> fp16 [D, 768], k = ky*48 + kx*3 + c (matches im2col_patch16)
  PK_NECK3,      // neck 3x3 conv [256,256,3,3] -> fp16 [256, 2304], k = tap*256 + c
  PK_CONVT,      // ConvTranspose2d(k=2,s=2) [cin, cout, 2, 2] -> fp16 [N = (d, co), K = ci] with d = di*2 + dj, so that
                 // output column block d is sub-pixel (di,dj) (SURVEY.md §8a P7)
  PK_TILE4,      // bias [cout] once per sub-pixel d -> fp32 [4, cout]
  PK_DEC4,       // map_decoder.7 [32, 2, 2, 2] -> fp32 [ci][d*2 + co]
  PK_PAIR_ST,    // pair_proj.weight [128, 258] -> fp16 [256, 128]: rows 0..127 Ws, 128..255 Wt
  PK_PAIR_OFF,   // pair_proj.weight [128, 258] -> fp32 [128, 2]: the two offset columns
};

bool packs_f16(int pack) {
  return pack == PK_F16 || pack == PK_PATCH || pack == PK_NECK3 || pack == PK_CONVT || pack == PK_PAIR_ST;
}

__global__ void pack_kernel(const float* __restrict__ src, int pack, int cin, int cout, long long n, float* d32,
                            __half* d16) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long j = i;
  switch (pack) {
    case PK_PATCH: {   // o[n*768 + ky*48 + kx*3 + c] = w[((n*3 + c)*16 + ky)*16 + kx]
      const long long k = i % 768, ky = k / 48, kx = k % 48 / 3, c = k % 3;
      j = ((i / 768 * 3 + c) * 16 + ky) * 16 + kx;
      break;
    }
    case PK_NECK3: {   // o[n*2304 + tap*256 + c] = w[(n*256 + c)*9 + tap]
      const long long k = i % 2304;
      j = (i / 2304 * 256 + k % 256) * 9 + k / 256;
      break;
    }
    case PK_CONVT: {   // o[(d*cout + co)*cin + ci] = w[(ci*cout + co)*4 + d]
      const long long ci = i % cin, dc = i / cin, co = dc % cout, d = dc / cout;
      j = (ci * cout + co) * 4 + d;
      break;
    }
    case PK_TILE4: j = i % cout; break;
    case PK_DEC4: {    // o[ci*8 + d*2 + co] = w[(ci*2 + co)*4 + d]
      const long long ci = i / 8, d = (i % 8) / 2, co = i % 2;
      j = (ci * 2 + co) * 4 + d;
      break;
    }
    case PK_PAIR_ST: {   // o[r*128 + k] = w[(r % 128)*258 + (r / 128)*128 + k]
      const long long r = i / 128, k = i % 128;
      j = (r % 128) * 258 + (r / 128) * 128 + k;
      break;
    }
    case PK_PAIR_OFF: j = (i / 2) * 258 + 256 + i % 2; break;
    default: break;
  }
  const float v = src[j];
  if (d16) d16[i] = __float2half_rn(v);
  else d32[i] = v;
}

// The regions of the handle's packed weights in the order samroad_finalize_weights allocates them: visit(region,
// field) with the handle member that holds the region's device address (a float* or __half* lvalue).  The blocks
// must exist with their windows set.
template <typename Visit>
void packed_regions(samroad_ctx* h, Visit&& visit) {
  const SamRoadCfg& c = h->cfg;
  const int64_t D = h->D, s = h->s, hd = h->hd;
  bool refresh = false;
  auto region = [&](auto& field, int pack, int64_t n, std::vector<Source> src, int cin = 0, int cout = 0,
                    HostStep host = HS_NONE) { visit(Region{pack, n, cin, cout, host, refresh, std::move(src)}, field); };
  auto copy = [&](auto& field, int pack, const std::string& key, std::vector<int64_t> shape) {
    int64_t n = 1;
    for (int64_t d : shape) n *= d;
    region(field, pack, n, {{key, std::move(shape), 0}});
  };
  auto f32 = [&](auto& field, const std::string& key, std::vector<int64_t> shape) {
    copy(field, PK_F32, key, std::move(shape));
  };
  auto f16 = [&](auto& field, const std::string& key, std::vector<int64_t> shape) {
    copy(field, PK_F16, key, std::move(shape));
  };
  auto convT = [&](auto& field, const std::string& key, int cin, int cout) {
    region(field, PK_CONVT, 4LL * cin * cout, {{key, {cin, cout, 2, 2}, 0}}, cin, cout);
  };
  auto tile4 = [&](auto& field, const std::string& key, int cout) {
    region(field, PK_TILE4, 4LL * cout, {{key, {cout}, 0}}, 0, cout);
  };

  // ---- image encoder ----
  region(h->pe_w, PK_PATCH, D * 768, {{"image_encoder.patch_embed.proj.weight", {D, 3, 16, 16}, 0}});
  f32(h->pe_b, "image_encoder.patch_embed.proj.bias", {D});
  f32(h->pos, "image_encoder.pos_embed", {1, s, s, D});
  for (int i = 0; i < c.depth; ++i) {
    BlockW& b = h->blocks[i];
    const std::string k = fmt_key("image_encoder.blocks.%d.", i);
    const int64_t rel_rows = 2 * b.win - 1;
    f32(b.ln1_g, k + "norm1.weight", {D});
    f32(b.ln1_b, k + "norm1.bias", {D});
    f32(b.ln2_g, k + "norm2.weight", {D});
    f32(b.ln2_b, k + "norm2.bias", {D});
    if (c.lora_rank > 0) {
      const int64_t r = c.lora_rank;
      const std::string q = k + "attn.qkv.";
      region(b.qkv_w, PK_F16, 3 * D * D,
             {{q + "weight", {3 * D, D}, 0}, {q + "linear_a_q.weight", {r, D}, 0}, {q + "linear_b_q.weight", {D, r}, 0},
              {q + "linear_a_v.weight", {r, D}, 0}, {q + "linear_b_v.weight", {D, r}, 0}},
             0, 0, HS_LORA_QKV);
    } else {
      f16(b.qkv_w, k + "attn.qkv.weight", {3 * D, D});
    }
    f32(b.qkv_b, k + "attn.qkv.bias", {3 * D});
    f16(b.proj_w, k + "attn.proj.weight", {D, D});
    f32(b.proj_b, k + "attn.proj.bias", {D});
    f32(b.rel_h, k + "attn.rel_pos_h", {rel_rows, hd});
    f32(b.rel_w, k + "attn.rel_pos_w", {rel_rows, hd});
    f16(b.lin1_w, k + "mlp.lin1.weight", {4 * D, D});
    f32(b.lin1_b, k + "mlp.lin1.bias", {4 * D});
    f16(b.lin2_w, k + "mlp.lin2.weight", {D, 4 * D});
    f32(b.lin2_b, k + "mlp.lin2.bias", {D});
  }
  // neck (image_encoder.py:88-104)
  f16(h->neck0_w, "image_encoder.neck.0.weight", {256, D, 1, 1});
  f32(h->neck1_g, "image_encoder.neck.1.weight", {256});
  f32(h->neck1_b, "image_encoder.neck.1.bias", {256});
  region(h->neck2_w, PK_NECK3, 256 * 2304, {{"image_encoder.neck.2.weight", {256, 256, 3, 3}, 0}});
  f32(h->neck3_g, "image_encoder.neck.3.weight", {256});
  f32(h->neck3_b, "image_encoder.neck.3.bias", {256});

  if (!c.use_sam_decoder) {
    // ---- naive map decoder (model.py:286-295) ----
    refresh = true;
    convT(h->dec1_w, "map_decoder.0.weight", 256, 128);
    tile4(h->dec1_b, "map_decoder.0.bias", 128);
    f32(h->dec_ln_g, "map_decoder.1.weight", {128});
    f32(h->dec_ln_b, "map_decoder.1.bias", {128});
    convT(h->dec2_w, "map_decoder.3.weight", 128, 64);
    tile4(h->dec2_b, "map_decoder.3.bias", 64);
    convT(h->dec3_w, "map_decoder.5.weight", 64, 32);
    f32(h->dec3_b, "map_decoder.5.bias", {32});
    region(h->dec4_w, PK_DEC4, 32 * 8, {{"map_decoder.7.weight", {32, 2, 2, 2}, 0}});
    f32(h->dec4_b, "map_decoder.7.bias", {2});
  } else {
    // ---- SAM mask decoder + null-prompt encoder (model.py:260-282) ----
    SamDecoderWeights& S = h->sam;
    const std::string md = "mask_decoder.", tr = "mask_decoder.transformer.";
    region(S.tokens, PK_F32, 4 * 256, {{md + "iou_token.weight", {1, 256}, 0}, {md + "mask_tokens.weight", {3, 256}, 256}});
    f32(S.no_mask_embed, "prompt_encoder.no_mask_embed.weight", {1, 256});
    region(S.dense_pe, PK_F32, s * s * 256,
           {{"prompt_encoder.pe_layer.positional_encoding_gaussian_matrix", {2, 128}, 0}}, 0, 0, HS_DENSE_PE);
    auto attn = [&](SamAttnW& a, const std::string& p, int64_t internal) {
      f32(a.qw, p + "q_proj.weight", {internal, 256}); f32(a.qb, p + "q_proj.bias", {internal});
      f32(a.kw, p + "k_proj.weight", {internal, 256}); f32(a.kb, p + "k_proj.bias", {internal});
      f32(a.vw, p + "v_proj.weight", {internal, 256}); f32(a.vb, p + "v_proj.bias", {internal});
      f32(a.ow, p + "out_proj.weight", {256, internal}); f32(a.ob, p + "out_proj.bias", {256});
    };
    for (int l = 0; l < 2; ++l) {
      const std::string p = tr + "layers." + std::to_string(l) + ".";
      attn(S.self_attn[l], p + "self_attn.", 256);
      attn(S.t2i[l], p + "cross_attn_token_to_image.", 128);
      attn(S.i2t[l], p + "cross_attn_image_to_token.", 128);
      f32(S.n1g[l], p + "norm1.weight", {256}); f32(S.n1b[l], p + "norm1.bias", {256});
      f32(S.n2g[l], p + "norm2.weight", {256}); f32(S.n2b[l], p + "norm2.bias", {256});
      f32(S.n3g[l], p + "norm3.weight", {256}); f32(S.n3b[l], p + "norm3.bias", {256});
      f32(S.n4g[l], p + "norm4.weight", {256}); f32(S.n4b[l], p + "norm4.bias", {256});
      f32(S.l1w[l], p + "mlp.lin1.weight", {2048, 256}); f32(S.l1b[l], p + "mlp.lin1.bias", {2048});
      f32(S.l2w[l], p + "mlp.lin2.weight", {256, 2048}); f32(S.l2b[l], p + "mlp.lin2.bias", {256});
      f16(S.t2i_kw16[l], p + "cross_attn_token_to_image.k_proj.weight", {128, 256});
      f16(S.t2i_vw16[l], p + "cross_attn_token_to_image.v_proj.weight", {128, 256});
      f16(S.i2t_qw16[l], p + "cross_attn_image_to_token.q_proj.weight", {128, 256});
      f16(S.i2t_ow16[l], p + "cross_attn_image_to_token.out_proj.weight", {256, 128});
    }
    attn(S.final_attn, tr + "final_attn_token_to_image.", 128);
    f16(S.t2i_kw16[2], tr + "final_attn_token_to_image.k_proj.weight", {128, 256});
    f16(S.t2i_vw16[2], tr + "final_attn_token_to_image.v_proj.weight", {128, 256});
    f32(S.nfg, tr + "norm_final_attn.weight", {256}); f32(S.nfb, tr + "norm_final_attn.bias", {256});
    for (int mi = 0; mi < 2; ++mi)
      for (int j = 0; j < 3; ++j) {
        const std::string k = md + "output_hypernetworks_mlps." + std::to_string(mi + 1) + ".layers." +
                              std::to_string(j) + ".";
        const int64_t out = j == 2 ? 32 : 256;
        f32(S.hw[mi][j], k + "weight", {out, 256});
        f32(S.hb[mi][j], k + "bias", {out});
      }
    convT(S.up1_w, md + "output_upscaling.0.weight", 256, 64);
    tile4(S.up1_b, md + "output_upscaling.0.bias", 64);
    f32(S.up1_g, md + "output_upscaling.1.weight", {64});
    f32(S.up1_beta, md + "output_upscaling.1.bias", {64});
    convT(S.up2_w, md + "output_upscaling.3.weight", 64, 32);
    tile4(S.up2_b, md + "output_upscaling.3.bias", 32);
  }

  // ---- TopoNet (model.py:61-86) ----
  refresh = true;
  f16(h->tp_feat_w, "topo_net.feature_proj.weight", {128, 256});
  f32(h->tp_feat_b, "topo_net.feature_proj.bias", {128});
  region(h->tp_st_w, PK_PAIR_ST, 256 * 128, {{"topo_net.pair_proj.weight", {128, 258}, 0}});
  region(h->tp_off_w, PK_PAIR_OFF, 128 * 2, {{"topo_net.pair_proj.weight", {128, 258}, 0}});
  f32(h->tp_pair_b, "topo_net.pair_proj.bias", {128});
  if (c.toponet_version != SAMROAD_TOPO_NO_TRANSFORMER) {
    std::vector<Source> chunks;   // tp_chunks: per layer Wq|Wk|Wv, Wo, W1, W2 as [128, 128] blocks
    for (int l = 0; l < 3; ++l) {
      const std::string k = fmt_key("topo_net.transformer_encoder.layers.%d.", l);
      const int64_t at = static_cast<int64_t>(l) * 6 * 128 * 128;
      chunks.push_back({k + "self_attn.in_proj_weight", {384, 128}, at});
      chunks.push_back({k + "self_attn.out_proj.weight", {128, 128}, at + 3 * 128 * 128});
      chunks.push_back({k + "linear1.weight", {128, 128}, at + 4 * 128 * 128});
      chunks.push_back({k + "linear2.weight", {128, 128}, at + 5 * 128 * 128});
    }
    region(h->tp_chunks, PK_F16, 18 * 128 * 128, std::move(chunks));
    for (int l = 0; l < 3; ++l) {
      TopoLayerParams& t = h->tp_layers[l];
      const std::string k = fmt_key("topo_net.transformer_encoder.layers.%d.", l);
      f32(t.in_b, k + "self_attn.in_proj_bias", {384});
      f32(t.out_b, k + "self_attn.out_proj.bias", {128});
      f32(t.l1_b, k + "linear1.bias", {128});
      f32(t.l2_b, k + "linear2.bias", {128});
      f32(t.n1_g, k + "norm1.weight", {128});
      f32(t.n1_b, k + "norm1.bias", {128});
      f32(t.n2_g, k + "norm2.weight", {128});
      f32(t.n2_b, k + "norm2.bias", {128});
    }
  }
  f32(h->tp_out_w, "topo_net.output_proj.weight", {1, 128});
  f32(h->tp_out_b, "topo_net.output_proj.bias", {1});
}

// Packs n_src fp32 values at src (device memory) into region r, whose storage starts at dst, from element `at`
// on; stream-ordered.  A copy writes n_src elements, every other packing the whole region.
int pack_source(const Region& r, const float* src, int64_t n_src, void* dst, int64_t at, cudaStream_t st) {
  const long long n = r.pack == PK_F32 || r.pack == PK_F16 ? n_src : r.n;
  const bool f16 = packs_f16(r.pack);
  SRB_LAUNCH(pack_kernel, blocks_for(n, 256), 256, 0, st, src, r.pack, r.cin, r.cout, n,
             f16 ? nullptr : static_cast<float*>(dst) + at, f16 ? static_cast<__half*>(dst) + at : nullptr);
  return 0;
}

// The fp32 values a region with a host step packs, computed from its sources' staged values.
std::vector<float> host_values(const samroad_ctx* h, const Region& r, const std::vector<const HostTensor*>& in) {
  const int64_t D = h->D, s = h->s;
  if (r.host == HS_LORA_QKV) {
    // qkv = xW^T + b ; q += B_q A_q x ; v += B_v A_v x   (model.py:179-186), merged into W in fp32
    const int64_t rank = h->cfg.lora_rank;
    const HostTensor *aq = in[1], *bq = in[2], *av = in[3], *bv = in[4];
    std::vector<float> wf = in[0]->data;
    for (int64_t n = 0; n < D; ++n)
      for (int64_t j = 0; j < rank; ++j) {
        const float bqv = bq->data[n * rank + j], bvv = bv->data[n * rank + j];
        float* wq = &wf[n * D];
        float* wv = &wf[(2 * D + n) * D];
        const float* aqr = &aq->data[j * D];
        const float* avr = &av->data[j * D];
        for (int64_t k = 0; k < D; ++k) {
          wq[k] += bqv * aqr[k];
          wv[k] += bvv * avr[k];
        }
      }
    return wf;
  }
  // HS_DENSE_PE: PromptEncoder.get_dense_pe (prompt_encoder.py:62-71,185-205), constant per config; on the host,
  // since the device sinf/cosf may differ in the last bit
  const std::vector<float>& G = in[0]->data;
  std::vector<float> pe(static_cast<size_t>(s) * s * 256);
  for (int y = 0; y < s; ++y)
    for (int x = 0; x < s; ++x) {
      const float cx = 2.0f * ((x + 0.5f) / s) - 1.0f, cy = 2.0f * ((y + 0.5f) / s) - 1.0f;
      for (int k = 0; k < 128; ++k) {
        const float a = 6.283185307179586f * (cx * G[k] + cy * G[128 + k]);
        pe[(static_cast<size_t>(y) * s + x) * 256 + k] = sinf(a);
        pe[(static_cast<size_t>(y) * s + x) * 256 + 128 + k] = cosf(a);
      }
    }
  return pe;
}

// samroad_finalize_weights' state: the first failure wins, and its message is kept.
struct Packer {
  samroad_ctx* h;
  bool ok = true;
  char msg[512] = "";
  DeviceBuffer scratch;   // the fp32 values being packed

  const HostTensor* get(const std::string& key, const std::vector<int64_t>& shape) {
    auto it = h->staged.find(key);
    if (it == h->staged.end()) {
      fail("missing state_dict key '%s'", key.c_str());
      return nullptr;
    }
    const HostTensor& t = it->second;
    if (t.shape != shape) {
      std::string got;
      for (auto d : t.shape) got += std::to_string(d) + ",";
      std::string want;
      for (auto d : shape) want += std::to_string(d) + ",";
      fail("state_dict key '%s' has shape [%s] but [%s] is required", key.c_str(), got.c_str(),
           want.c_str());
      return nullptr;
    }
    return &t;
  }
  void fail(const char* fmt, ...) {
    if (!ok) return;
    ok = false;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(msg, sizeof(msg), fmt, ap);
    va_end(ap);
  }
  // one device buffer per region, with 256 bytes of tail slack
  void* alloc(size_t bytes) {
    if (!ok) return nullptr;
    DeviceBuffer d;
    if (d.reserve(bytes + 256, "samroad_finalize_weights")) {
      fail("cudaMalloc of %zu bytes for weights failed", bytes);
      return nullptr;
    }
    void* p = d.get();
    h->weight_allocs.push_back(std::move(d));
    return p;
  }
  // uploads v into the scratch buffer and packs it into region r at dst, on the legacy default stream
  void pack(const Region& r, const std::vector<float>& v, void* dst, int64_t at) {
    if (!ok) return;
    const size_t bytes = v.size() * sizeof(float);
    if (grow(scratch, bytes, "samroad_finalize_weights") != 0) {
      fail("%s", get_last_error());
    } else if (cudaMemcpy(scratch.get(), v.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
      fail("cudaMemcpy of weights failed");
    } else if (pack_source(r, scratch.as<float>(), static_cast<int64_t>(v.size()), dst, at, nullptr) != 0) {
      fail("%s", get_last_error());
    }
  }
};

// ---- activation workspace layout for the encoder + decoder ------------------------------------------
struct EncWs {
  float* X;        // [M, D]   residual stream (fp32)
  __half* XN;      // [M, max(D,768)] LN output / patch im2col / fp16 copy of X
  __half* QKV;     // [M, 3D]
  __half* ATT;     // [M, D]
  __half* H;       // [M, 4D]  MLP hidden; reused: IM2 [M, 2304], D2 [4M, 256]
  __half* N1;      // [M, 256] neck conv1 + LN ; reused: D1 [M, 512] needs 2x -> own buffer below
  __half* FEAT;    // [M, 256] neck output (fp16 NHWC)
  __half* D1;      // [M, 512]
  uint8_t* RGB;    // [B, P, P, 3] uint8 tiles cropped from a scene (samroad_encode_masks_scene)
  size_t total;
};

EncWs layout_enc(const samroad_ctx* h, int B, void* base) {
  const size_t M = static_cast<size_t>(B) * h->T, D = h->D;
  Layout L(base, 1024);
  EncWs w;
  w.X = L.take<float>(M * D);
  w.XN = L.take<__half>(M * (D > 768 ? D : 768));
  w.QKV = L.take<__half>(M * 3 * D);
  w.ATT = L.take<__half>(M * D);
  w.H = L.take<__half>(M * 4 * D);   // >= M*2304 and >= 4M*256 for D >= 768
  w.N1 = L.take<__half>(M * 256);
  w.FEAT = L.take<__half>(M * 256);
  w.D1 = L.take<__half>(M * 512);
  w.RGB = L.take<uint8_t>(M * 768);    // B * P * P * 3 = M * 256 * 3
  w.total = L.bytes();
  return w;
}

// samroad_op_encoder_taps: copy a workspace tensor into a caller's buffer (NULL: not requested) before
// a later launch reuses that workspace
int tap_copy(void* dst, const void* src, size_t bytes, cudaStream_t st) {
  if (dst) SRB_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st));
  return 0;
}

struct TopoWs {
  __half* F16;     // [B*N, 256]
  __half* PF16;    // [B*N, 128]
  float* PST;      // [B*N, 256]
  uint8_t* VF;     // [rows*Np]
  float* X32;      // [tok, 128]
  __half* X16;     // [tok, 128]
  __half* QKV16;   // [tok, 384]
  __half* ATT16;   // [tok, 128]
  __half* H16;     // [tok, 128]
  size_t total;
};

TopoWs layout_topo(int B, int N, int Ns, int Np, void* base) {
  const size_t pts = static_cast<size_t>(B) * N, tok = static_cast<size_t>(B) * Ns * Np;
  Layout L(base, 1024);
  TopoWs w;
  w.F16 = L.take<__half>(pts * 256);
  w.PF16 = L.take<__half>(pts * 128);
  w.PST = L.take<float>(pts * 256);
  w.VF = L.take<uint8_t>(tok);
  w.X32 = L.take<float>(tok * 128);
  w.X16 = L.take<__half>(tok * 128);
  w.QKV16 = L.take<__half>(tok * 384);
  w.ATT16 = L.take<__half>(tok * 128);
  w.H16 = L.take<__half>(tok * 128);
  w.total = L.bytes();
  return w;
}

// run a launcher with optional CUDA-event timing under a kernel-class tag
#define SRB_T(tag, flops, bytes, expr)                                   \
  do {                                                                   \
    h->timer.begin((tag), (double)(flops), (double)(bytes), st);         \
    int _rc = (expr);                                                    \
    h->timer.end(st);                                                    \
    if (_rc != 0) return _rc;                                            \
  } while (0)

int check_handle(samroad_handle_t h, bool need_weights) {
  SRB_REQUIRE(h != nullptr, "null samroad handle");
  SRB_REQUIRE(!need_weights || h->finalized,
              "weights not finalized: call samroad_load_tensor for every state_dict key, then "
              "samroad_finalize_weights");
  SRB_CUDA_OK(cudaSetDevice(h->device));
  return 0;
}

}  // namespace

// =================================================================================================
// lifetime
// =================================================================================================
extern "C" int samroad_create(const SamRoadCfg* cfg, int device, samroad_handle_t* out) {
  SRB_REQUIRE(cfg && out, "samroad_create: null argument");
  SRB_REQUIRE(cfg->patch_size > 0 && cfg->patch_size % 16 == 0 && cfg->patch_size <= 1024,
              "PATCH_SIZE=%d must be a multiple of 16 in (0,1024]", cfg->patch_size);
  SRB_REQUIRE(cfg->embed_dim % 128 == 0 && cfg->embed_dim >= 768 && cfg->embed_dim <= 1280,
              "embed_dim=%d unsupported", cfg->embed_dim);
  SRB_REQUIRE(cfg->num_heads > 0 && cfg->embed_dim % cfg->num_heads == 0,
              "embed_dim=%d not divisible by num_heads=%d", cfg->embed_dim, cfg->num_heads);
  const int hd = cfg->embed_dim / cfg->num_heads;
  SRB_REQUIRE(hd == 64 || hd == 80, "head_dim=%d unsupported (64 or 80)", hd);
  SRB_REQUIRE(cfg->depth > 0 && cfg->depth <= 64, "depth=%d unsupported", cfg->depth);
  SRB_REQUIRE(cfg->window_size > 0, "window_size=%d must be positive", cfg->window_size);
  SRB_TRY(open_device(device));
  cudaDeviceProp prop;
  SRB_CUDA_OK(cudaGetDeviceProperties(&prop, device));
  SRB_REQUIRE(prop.major == 9 && prop.minor == 0, "device %d is sm_%d%d; this library is built for sm_90a only",
              device, prop.major, prop.minor);
  samroad_ctx* h = new samroad_ctx();
  h->cfg = *cfg;
  h->device = device;
  h->s = cfg->patch_size / 16;
  h->T = h->s * h->s;
  h->D = cfg->embed_dim;
  h->hd = hd;
  *out = h;
  return 0;
}

extern "C" int samroad_destroy(samroad_handle_t h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  if (h->s_compute) { cudaStreamDestroy(h->s_h2d); cudaStreamDestroy(h->s_compute); cudaStreamDestroy(h->s_copy); }
  for (auto& sl : h->slots)
    for (cudaEvent_t e : {sl.ev_h2d, sl.ev_emb, sl.ev_scores, sl.ev_compute, sl.ev_done})
      if (e) cudaEventDestroy(e);
  delete h;
  return 0;
}

extern "C" int samroad_load_tensor(samroad_handle_t h, const char* key, const float* host_data,
                                   const int64_t* shape, int ndim) {
  SRB_REQUIRE(h && key && host_data && (shape || ndim == 0), "samroad_load_tensor: null argument");
  SRB_REQUIRE(ndim >= 0 && ndim <= 8, "samroad_load_tensor: ndim=%d", ndim);
  HostTensor t;
  t.shape.assign(shape, shape + ndim);
  const int64_t n = t.numel();
  SRB_REQUIRE(n >= 0, "samroad_load_tensor: negative size for '%s'", key);
  t.data.assign(host_data, host_data + n);
  h->staged[key] = std::move(t);
  h->finalized = false;
  return 0;
}

extern "C" int samroad_finalize_weights(samroad_handle_t h) {
  SRB_TRY(check_handle(h, false));
  // drop previously packed weights (re-load after load_state_dict); until this call succeeds the handle has none
  h->finalized = false;
  SRB_CUDA_OK(cudaDeviceSynchronize());
  h->refresh_targets.clear();
  h->weight_allocs.clear();

  Packer P{h};
  const SamRoadCfg& c = h->cfg;
  h->blocks.assign(c.depth, BlockW{});
  for (int i = 0; i < c.depth; ++i) {
    // A window block keeps its window size even when it exceeds the grid (s < 14, PATCH_SIZE < 224):
    // the s x s tokens are then padded to one window, whose pad tokens are softmax keys
    // (image_encoder.py:168-172), and the rel-pos tables have 2*window-1 rows.
    const bool glob = is_global_block(c, i);
    h->blocks[i].win = glob ? h->s : c.window_size;
    if (!glob && c.window_size > 64) P.fail("window_size=%d unsupported (at most 64)", c.window_size);
  }
  packed_regions(h, [&](const Region& r, auto& field) {
    std::vector<const HostTensor*> in;
    for (const Source& src : r.src) in.push_back(P.get(src.key, src.shape));
    void* dst = P.alloc(r.n * (packs_f16(r.pack) ? sizeof(__half) : sizeof(float)));
    if (!dst) return;
    field = static_cast<std::remove_reference_t<decltype(field)>>(dst);
    if (r.refresh)
      for (const Source& src : r.src) h->refresh_targets[src.key].push_back({r, dst, src});
    if (r.host != HS_NONE) {
      P.pack(r, host_values(h, r, in), dst, 0);
    } else {
      for (size_t i = 0; i < in.size(); ++i) P.pack(r, in[i]->data, dst, r.src[i].at);
    }
  });
  if (c.use_sam_decoder) {   // constant part of the decoder: layer-0 queries
    if (float* q0 = static_cast<float*>(P.alloc(4 * 256 * sizeof(float)))) {
      if (sam_decoder_prepare(h->sam, q0, nullptr) != 0 || cudaStreamSynchronize(nullptr) != cudaSuccess)
        P.fail("sam_decoder_prepare failed: %s", get_last_error());
      h->sam.q0 = q0;
    }
  }
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) P.fail("packing the weights failed: %s", cudaGetErrorString(e));

  if (!P.ok) {
    set_last_error("samroad_finalize_weights: %s", P.msg);
    return 3;
  }
  h->staged.clear();
  h->finalized = true;
  return 0;
}

// Used by train.cu: the tile size and head variants of a handle.
int samroad_handle_head_config(samroad_handle_t h, int* patch_size, int* toponet_version, int* use_sam_decoder) {
  SRB_TRY(check_handle(h, true));
  *patch_size = h->cfg.patch_size;
  *toponet_version = h->cfg.toponet_version;
  *use_sam_decoder = h->cfg.use_sam_decoder;
  return 0;
}

extern "C" int samroad_update_tensor_device(samroad_handle_t h, const char* key, const float* dev_data,
                                            const int64_t* shape, int ndim, void* stream) {
  SRB_TRY(check_handle(h, true));
  SRB_REQUIRE(key && dev_data && (shape || ndim == 0) && ndim >= 0 && ndim <= 8,
              "samroad_update_tensor_device: bad arguments");
  SRB_REQUIRE(!h->cfg.use_sam_decoder, "samroad_update_tensor_device: the SAM mask decoder is repacked on the host only");
  const auto it = h->refresh_targets.find(key);
  SRB_REQUIRE(it != h->refresh_targets.end(),
              "samroad_update_tensor_device: '%s' is not a head tensor of this configuration", key);
  const std::vector<RefreshTarget>& tg = it->second;
  const std::vector<int64_t>& want = tg[0].src.shape;
  SRB_REQUIRE(want == std::vector<int64_t>(shape, shape + ndim), "samroad_update_tensor_device: '%s' has the wrong shape",
              key);
  int64_t n = 1;
  for (int64_t d : want) n *= d;
  for (const RefreshTarget& t : tg)
    SRB_TRY(pack_source(t.r, dev_data, n, t.dst, t.src.at, static_cast<cudaStream_t>(stream)));
  return 0;
}

// =================================================================================================
// encoder + mask head
// =================================================================================================
extern "C" size_t samroad_workspace_bytes(samroad_handle_t h, int B) {
  if (!h || B <= 0) return 0;
  return layout_enc(h, B, nullptr).total;
}

extern "C" int samroad_encode_masks(samroad_handle_t h, const void* rgb, int rgb_dtype, int B,
                                    float* mask_scores, float* mask_logits,
                                    float* image_embeddings, void* stream) {
  SRB_TRY(check_handle(h, true));
  SRB_REQUIRE(rgb && image_embeddings, "samroad_encode_masks: null rgb / image_embeddings");
  SRB_REQUIRE(rgb_dtype == SAMROAD_F32 || rgb_dtype == SAMROAD_U8,
              "samroad_encode_masks: rgb dtype %d (want SAMROAD_F32 or SAMROAD_U8)", rgb_dtype);
  if (B <= 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int T = h->T, D = h->D, s = h->s, P = h->cfg.patch_size;
  const long Ml = static_cast<long>(B) * T;
  SRB_REQUIRE(Ml * 16 < 2147483647L, "batch of %d tiles is too large for one call", B);
  const int M = static_cast<int>(Ml);
  SRB_TRY(grow(h->ws, layout_enc(h, B, nullptr).total, "samroad_encode_masks"));
  EncWs w = layout_enc(h, B, h->ws.get());

  // patch embed + pos embed  (image_encoder.py:107-109, 387-395; normalisation model.py:465-467)
  const float inv_std[3] = {1.0f / kPixelStd[0], 1.0f / kPixelStd[1], 1.0f / kPixelStd[2]};
  const double Md = M, Dd = D;
  const double px_bytes = static_cast<double>(B) * P * P * 3 * (rgb_dtype == SAMROAD_U8 ? 1 : 4);
  SRB_T(KT_PATCH_IM2COL, 0, px_bytes + Md * 768 * 2,
        im2col_patch16(rgb, rgb_dtype == SAMROAD_U8 ? 1 : 0, B, P, kPixelMean, inv_std, w.XN, st));
  SRB_T(KT_GEMM_PATCH, 2 * Md * Dd * 768, Md * 768 * 2 + Md * Dd * 4,
        gemm_f32out(w.XN, 768, h->pe_w, 768, M, D, 768, h->pe_b, nullptr, h->pos, T, w.X, D, st));
  const SamroadEncoderTaps* tp = h->taps;
  const size_t MD = static_cast<size_t>(M) * D;
  if (tp) SRB_TRY(tap_copy(tp->tokens0, w.X, MD * 4, st));

  // transformer blocks (image_encoder.py:166-182).  Both LayerNorms of block i walk the token rows
  // descending when i is even and ascending when i is odd (all ascending under the test hook); the
  // effect of this order on L2 reuse has not been measured on the H100.
  for (int i = 0; i < h->cfg.depth; ++i) {
    const BlockW& b = h->blocks[i];
    const bool ln_reverse = i % 2 == 0 && !g_ln_ascending;
    // algorithmic attention FLOPs: real query/key tokens only (SURVEY.md §8d)
    double att_flops = 0;
    {
      const int nw = (s + b.win - 1) / b.win;
      for (int wy = 0; wy < nw; ++wy)
        for (int wx = 0; wx < nw; ++wx) {
          const double ry = (wy + 1) * b.win <= s ? b.win : s - wy * b.win;
          const double rx = (wx + 1) * b.win <= s ? b.win : s - wx * b.win;
          att_flops += 4.0 * (ry * rx) * (ry * rx) * h->hd;
        }
      att_flops *= static_cast<double>(B) * h->cfg.num_heads;
    }
    const bool det = tp && tp->detail_block == i;
    SRB_T(KT_LAYERNORM, 0, Md * Dd * 6, layernorm_f16(w.X, b.ln1_g, b.ln1_b, 1e-6f, M, D, w.XN, ln_reverse, st));
    if (det) SRB_TRY(tap_copy(tp->ln1, w.XN, MD * 2, st));
    SRB_T(KT_GEMM_QKV, 2 * Md * 3 * Dd * Dd, Md * Dd * 2 + Md * 3 * Dd * 2,
          gemm_f16out(w.XN, D, b.qkv_w, D, M, 3 * D, D, b.qkv_b, ACT_NONE, w.QKV, 3 * D, st));
    if (det) SRB_TRY(tap_copy(tp->qkv, w.QKV, MD * 6, st));
    SRB_T(b.win == s ? KT_ATTN_GLOBAL : KT_ATTN_WINDOW, att_flops, Md * 4 * Dd * 2,
          encoder_attention(w.QKV, b.qkv_b, b.rel_h, b.rel_w, B, s, b.win,
                            h->cfg.num_heads, h->hd, w.ATT, st));
    if (det) SRB_TRY(tap_copy(tp->att, w.ATT, MD * 2, st));
    SRB_T(KT_GEMM_PROJ, 2 * Md * Dd * Dd, Md * Dd * 2 + Md * Dd * 8,
          gemm_f32out(w.ATT, D, b.proj_w, D, M, D, D, b.proj_b, w.X, nullptr, 0, w.X, D, st));
    if (det) SRB_TRY(tap_copy(tp->x_attn, w.X, MD * 4, st));
    SRB_T(KT_LAYERNORM, 0, Md * Dd * 6, layernorm_f16(w.X, b.ln2_g, b.ln2_b, 1e-6f, M, D, w.XN, ln_reverse, st));
    if (det) SRB_TRY(tap_copy(tp->ln2, w.XN, MD * 2, st));
    SRB_T(KT_GEMM_LIN1, 2 * Md * 4 * Dd * Dd, Md * Dd * 2 + Md * 4 * Dd * 2,
          gemm_f16out(w.XN, D, b.lin1_w, D, M, 4 * D, D, b.lin1_b, ACT_GELU, w.H, 4 * D, st));
    if (det) SRB_TRY(tap_copy(tp->h, w.H, MD * 8, st));
    SRB_T(KT_GEMM_LIN2, 2 * Md * 4 * Dd * Dd, Md * 4 * Dd * 2 + Md * Dd * 8,
          gemm_f32out(w.H, 4 * D, b.lin2_w, 4 * D, M, D, 4 * D, b.lin2_b, w.X, nullptr, 0, w.X, D,
                      st));
    if (tp && tp->blocks && (tp->block_mask >> i & 1)) {
      const int slot = __builtin_popcountll(tp->block_mask & ((uint64_t{1} << i) - 1));
      SRB_TRY(tap_copy(tp->blocks + slot * MD, w.X, MD * 4, st));
    }
  }

  // neck (image_encoder.py:88-104,114): 1x1 conv -> LN2d -> 3x3 conv -> LN2d
  SRB_T(KT_NECK, 0, Md * Dd * 6, convert_f32_f16(w.X, static_cast<long>(M) * D, w.XN, st));
  SRB_T(KT_NECK, 2 * Md * 256 * Dd, Md * Dd * 2 + Md * 256 * 2,
        gemm_ln(w.XN, D, h->neck0_w, D, M, 256, D, nullptr, nullptr, h->neck1_g, h->neck1_b, 1e-6f,
                256, ACT_NONE, w.N1, nullptr, nullptr, T, 256, st));
  if (tp) SRB_TRY(tap_copy(tp->n1, w.N1, static_cast<size_t>(M) * 256 * 2, st));
  if (128 % s == 0 && T % 128 == 0) {
    // 3x3 conv as an implicit GEMM: the TMA producer reads the nine tap-shifted slabs of the NHWC
    // tensor directly (zero fill outside the image), no im2col buffer
    SRB_T(KT_NECK, 2 * Md * 256 * 2304, Md * 256 * 2 * 9 + Md * 256 * 6,
          gemm_ln(w.N1, 256, h->neck2_w, 2304, M, 256, 2304, nullptr, nullptr, h->neck3_g, h->neck3_b,
                  1e-6f, 256, ACT_NONE, w.FEAT, nullptr, image_embeddings, T, 256, st, s));
  } else {
    __half* IM2 = w.H;
    SRB_T(KT_NECK, 0, Md * 256 * 2 * 10, im2col_3x3(w.N1, B, s, 256, IM2, st));
    SRB_T(KT_NECK, 2 * Md * 256 * 2304, Md * 2304 * 2 + Md * 256 * 6,
          gemm_ln(IM2, 2304, h->neck2_w, 2304, M, 256, 2304, nullptr, nullptr, h->neck3_g, h->neck3_b,
                  1e-6f, 256, ACT_NONE, w.FEAT, nullptr, image_embeddings, T, 256, st));
  }
  if (tp) SRB_TRY(tap_copy(tp->feat16, w.FEAT, static_cast<size_t>(M) * 256 * 2, st));

  // naive map decoder (model.py:286-295, 490-491) as three GEMMs, pixel shuffle by row indexing
  if (h->ev_emb_hook) SRB_CUDA_OK(cudaEventRecord(h->ev_emb_hook, st));   // embeddings are final here
  if ((mask_scores || mask_logits) && h->cfg.use_sam_decoder) {
    // SAM mask decoder (model.py:471-488): null prompts, TwoWayTransformer, upscaler, x4 bilinear
    SRB_TRY(grow(h->sam_ws, sam_decoder_ws_bytes(B, T), "samroad_encode_masks"));
    SRB_T(KT_DECODER, 0.91e9 * B, Md * 256 * 4 * 10,
          sam_decoder_forward(h->sam, image_embeddings, B, s, P, h->sam_ws.get(), mask_scores, mask_logits, st));
  } else if (mask_scores || mask_logits) {
    SRB_T(KT_DECODER, 2 * Md * 512 * 256, Md * 256 * 2 + Md * 512 * 2,
          gemm_ln(w.FEAT, 256, h->dec1_w, 256, M, 512, 256, h->dec1_b, nullptr, h->dec_ln_g,
                  h->dec_ln_b, 1e-6f, 128, ACT_GELU, w.D1, nullptr, nullptr, T, 512, st));
    if (tp) SRB_TRY(tap_copy(tp->d1, w.D1, static_cast<size_t>(M) * 512 * 2, st));
    __half* D2 = w.H;
    SRB_T(KT_DECODER, 2 * Md * 4 * 256 * 128, Md * 512 * 2 + Md * 1024 * 2,
          gemm_f16out(w.D1, 128, h->dec2_w, 128, 4 * M, 256, 128, h->dec2_b, ACT_GELU, D2, 256, st));
    if (tp) SRB_TRY(tap_copy(tp->d2, D2, static_cast<size_t>(M) * 1024 * 2, st));
    SRB_T(KT_DECODER, 2 * Md * 16 * (128 * 64 + 4 * 32 * 8), Md * 1024 * 2 + Md * 512 * 4,
          gemm_dec_final(D2, 64, h->dec3_w, 64, 16 * M, 64, h->dec3_b, h->dec4_w, h->dec4_b, s, P,
                         mask_scores, mask_logits, st));
  }
  return 0;
}

// Tiles addressed inside a uint8 scene that already lives on the device (inferencer.py:43-58,87-96
// without the per-tile host crops and the synchronous float32 upload): crop on the device, then the
// same path as samroad_encode_masks.
extern "C" int samroad_encode_masks_scene(samroad_handle_t h, const uint8_t* scene, int H, int W,
                                          const int32_t* tile_xy, int B, float* mask_scores,
                                          float* mask_logits, float* image_embeddings, void* stream) {
  SRB_TRY(check_handle(h, true));
  SRB_REQUIRE(scene && tile_xy && image_embeddings, "samroad_encode_masks_scene: null argument");
  if (B <= 0) return 0;
  const int P = h->cfg.patch_size;
  SRB_REQUIRE(H >= P && W >= P, "samroad_encode_masks_scene: scene %dx%d smaller than a %d tile", H, W, P);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SRB_TRY(grow(h->ws, layout_enc(h, B, nullptr).total, "samroad_encode_masks_scene"));
  EncWs w = layout_enc(h, B, h->ws.get());
  SRB_T(KT_PATCH_IM2COL, 0, 2.0 * B * P * P * 3, crop_tiles(scene, H, W, tile_xy, B, P, w.RGB, st));
  return samroad_encode_masks(h, w.RGB, SAMROAD_U8, B, mask_scores, mask_logits, image_embeddings, stream);
}

extern "C" int samroad_encode_masks_host(samroad_handle_t h, const void* rgb_host, int rgb_dtype,
                                         int B, float* mask_scores_host,
                                         float* image_embeddings_host) {
  return samroad_infer_batch_host(h, rgb_host, rgb_dtype, B, nullptr, 0, nullptr, 0, nullptr, 0, 0, 0,
                                  mask_scores_host, image_embeddings_host, nullptr);
}

// =================================================================================================
// TopoNet
// =================================================================================================
extern "C" int samroad_toponet(samroad_handle_t h, const float* image_embeddings,
                               const void* points, int pts_dtype, const void* pairs,
                               int pairs_dtype, const uint8_t* valid, int B, int N, int Ns, int Np,
                               float* topo_logits, float* topo_scores, void* stream) {
  SRB_TRY(check_handle(h, true));
  SRB_REQUIRE(image_embeddings && points && pairs && valid, "samroad_toponet: null input");
  SRB_REQUIRE(pts_dtype == SAMROAD_F32 || pts_dtype == SAMROAD_I64 || pts_dtype == SAMROAD_I32,
              "samroad_toponet: points dtype %d", pts_dtype);
  SRB_REQUIRE(pairs_dtype == SAMROAD_I64 || pairs_dtype == SAMROAD_I32,
              "samroad_toponet: pairs dtype %d", pairs_dtype);
  SRB_REQUIRE(Np >= 1 && Np <= 32, "samroad_toponet: n_pairs=%d must be in 1..32", Np);
  if (B <= 0 || Ns <= 0) return 0;
  SRB_REQUIRE(N > 0, "samroad_toponet: N=%d points but Ns=%d samples", N, Ns);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long tokl = static_cast<long>(B) * Ns * Np;
  SRB_REQUIRE(tokl < 2147483647L / 4, "samroad_toponet: %ld pair tokens is too many for one call",
              tokl);
  const int tok = static_cast<int>(tokl), pts = B * N, rows = B * Ns;
  SRB_TRY(grow(h->topo_ws, layout_topo(B, N, Ns, Np, nullptr).total, "samroad_toponet"));
  TopoWs w = layout_topo(B, N, Ns, Np, h->topo_ws.get());
  const int zero_off = h->cfg.toponet_version == SAMROAD_TOPO_NO_OFFSET;
  const bool no_tf = h->cfg.toponet_version == SAMROAD_TOPO_NO_TRANSFORMER;

  const double ptsd = pts, tokd = tok;
  SRB_T(KT_TOPO_SAMPLE, 0, ptsd * 256 * (16 + 2),
        topo_sample_features(image_embeddings, B, 256, h->s, h->cfg.patch_size, points, pts_dtype, N,
                             w.F16, st));
  SRB_T(KT_TOPO_GEMM, 2 * ptsd * 128 * 256, ptsd * 384 * 2,
        gemm_f16out(w.F16, 256, h->tp_feat_w, 256, pts, 128, 256, h->tp_feat_b, ACT_RELU, w.PF16, 128,
                    st));
  SRB_T(KT_TOPO_GEMM, 2 * ptsd * 256 * 128, ptsd * (256 + 1024),
        gemm_f32out(w.PF16, 128, h->tp_st_w, 128, pts, 256, 128, nullptr, nullptr, nullptr, 0, w.PST,
                    256, st));
  SRB_T(KT_TOPO_PAIR, 0, tokd * 2, topo_fix_valid(valid, rows, Np, w.VF, st));
  const bool fused = !no_tf && (Np == 16 || Np == 32);
  const TopoPairInputs pin{w.PST, h->tp_off_w, h->tp_pair_b, points, pairs, pts_dtype, pairs_dtype, N,
                           Ns * Np, zero_off};
  if (fused) {
    // all three encoder layers + output_proj in one persistent wgmma kernel
    SRB_T(KT_TOPO_GEMM, tokd * 2 * 128 * (384 + 128 * 3) * 3 + tokd * 4 * Np * 128 * 3 + tokd * 128 * 6,
          tokd * 1024 * 2 + tokd * 8,
          topo_transformer_fused(pin, h->tp_chunks, h->tp_layers, h->tp_out_w, h->tp_out_b, w.VF, tok, Np,
                                 topo_logits, topo_scores, st));
    return 0;
  }
  SRB_T(KT_TOPO_PAIR, tokd * 128 * 6, tokd * 128 * (8 + 6), topo_pair_features(pin, tok, w.X32, w.X16, st));
  if (!no_tf) {
    for (int l = 0; l < 3; ++l) {
      const TopoLayerParams& t = h->tp_layers[l];
      // this layer's [Wq|Wk|Wv], Wo, W1, W2 in tp_chunks
      const __half* in_w = h->tp_chunks + static_cast<size_t>(l) * 6 * 128 * 128;
      const __half* out_w = in_w + 3 * 128 * 128;
      const __half* l1_w = in_w + 4 * 128 * 128;
      const __half* l2_w = in_w + 5 * 128 * 128;
      SRB_T(KT_TOPO_GEMM, 2 * tokd * 384 * 128, tokd * 512 * 2,
            gemm_f16out(w.X16, 128, in_w, 128, tok, 384, 128, t.in_b, ACT_NONE, w.QKV16, 384, st));
      SRB_T(KT_TOPO_ATTN, 4 * tokd * Np * 128, tokd * 512 * 2,
            topo_attention(w.QKV16, w.VF, rows, Np, w.ATT16, st));
      SRB_T(KT_TOPO_GEMM, 2 * tokd * 128 * 128, tokd * 128 * (2 + 4 + 4 + 2),
            gemm_ln(w.ATT16, 128, out_w, 128, tok, 128, 128, t.out_b, w.X32, t.n1_g, t.n1_b, 1e-5f,
                    128, ACT_NONE, w.X16, w.X32, nullptr, 1, 128, st));
      SRB_T(KT_TOPO_GEMM, 2 * tokd * 128 * 128, tokd * 128 * 4,
            gemm_f16out(w.X16, 128, l1_w, 128, tok, 128, 128, t.l1_b, ACT_RELU, w.H16, 128, st));
      SRB_T(KT_TOPO_GEMM, 2 * tokd * 128 * 128, tokd * 128 * (2 + 4 + 4 + 2),
            gemm_ln(w.H16, 128, l2_w, 128, tok, 128, 128, t.l2_b, w.X32, t.n2_g, t.n2_b, 1e-5f, 128,
                    ACT_NONE, w.X16, w.X32, nullptr, 1, 128, st));
    }
  }
  SRB_T(KT_TOPO_OUT, 2 * tokd * 128, tokd * (512 + 8),
        topo_output(w.X32, no_tf ? nullptr : w.VF, h->tp_out_w, h->tp_out_b, tok, topo_logits,
                    topo_scores, st));
  return 0;
}

// =================================================================================================
// misc C ABI
// =================================================================================================
extern "C" int samroad_fuse_masks(const float* scores, int n_tiles, int P, const int32_t* tile_x0,
                                  const int32_t* tile_y0, int H, int W, uint8_t* keypoint_u8,
                                  uint8_t* road_u8, void* stream) {
  SRB_REQUIRE(scores && tile_x0 && tile_y0 && keypoint_u8 && road_u8, "samroad_fuse_masks: null");
  return fuse_masks(scores, n_tiles, P, tile_x0, tile_y0, H, W, keypoint_u8, road_u8,
                    static_cast<cudaStream_t>(stream));
}

extern "C" int samroad_timing_enable(samroad_handle_t h, int on) {
  SRB_REQUIRE(h != nullptr, "null samroad handle");
  SRB_CUDA_OK(cudaSetDevice(h->device));
  SRB_CUDA_OK(cudaDeviceSynchronize());
  h->timer.reset();
  h->timer.on = on != 0;
  return 0;
}

// Writes one JSON object {"<kernel class>": {"launches": n, "ms": total, "flops": f, "bytes": b}, ...}
// for everything recorded since samroad_timing_enable(h, 1); synchronises the device.
extern "C" int samroad_timing_read(samroad_handle_t h, char* buf, size_t cap) {
  SRB_REQUIRE(h != nullptr && buf != nullptr && cap > 2, "samroad_timing_read: bad arguments");
  SRB_CUDA_OK(cudaSetDevice(h->device));
  SRB_CUDA_OK(cudaDeviceSynchronize());
  double ms[KT_COUNT] = {0}, fl[KT_COUNT] = {0}, by[KT_COUNT] = {0};
  long cnt[KT_COUNT] = {0};
  for (const auto& r : h->timer.recs) {
    float t = 0.f;
    SRB_CUDA_OK(cudaEventElapsedTime(&t, r.a, r.b));
    ms[r.tag] += t; fl[r.tag] += r.flops; by[r.tag] += r.bytes; cnt[r.tag] += 1;
  }
  size_t off = 0;
  off += snprintf(buf + off, cap - off, "{");
  bool first = true;
  for (int t = 0; t < KT_COUNT && off + 200 < cap; ++t) {
    if (cnt[t] == 0) continue;
    off += snprintf(buf + off, cap - off,
                    "%s\"%s\": {\"launches\": %ld, \"ms\": %.6f, \"flops\": %.6e, \"bytes\": %.6e}",
                    first ? "" : ", ", kTagNames[t], cnt[t], ms[t], fl[t], by[t]);
    first = false;
  }
  snprintf(buf + off, cap - off, "}");
  return 0;
}

// One whole batch with HOST buffers, asynchronously, on staging slot 0 or 1: H2D of the tiles (+ TopoNet
// inputs) on an upload stream, encoder + mask head + TopoNet on the compute stream, D2H of image
// embeddings / mask scores / topology scores on a download stream as soon as each is final.  With two
// slots in flight the downloads of step i (202 MB at the bench workload) run under the upload and
// the compute of step i+1.  Any output may be NULL; TopoNet is skipped when points_host is NULL.
extern "C" int samroad_infer_batch_host_async(samroad_handle_t h, int slot, const void* rgb_host,
                                              int rgb_dtype, int B, const void* points_host,
                                              int pts_dtype, const void* pairs_host, int pairs_dtype,
                                              const uint8_t* valid_host, int N, int Ns, int Np,
                                              float* mask_scores_host, float* image_embeddings_host,
                                              float* topo_scores_host) {
  SRB_TRY(check_handle(h, true));
  SRB_REQUIRE(rgb_host, "samroad_infer_batch_host: null rgb");
  SRB_REQUIRE(slot == 0 || slot == 1, "samroad_infer_batch_host_async: slot %d (want 0 or 1)", slot);
  if (B <= 0) return 0;
  const size_t P = h->cfg.patch_size, s = h->s;
  const size_t in_bytes = static_cast<size_t>(B) * P * P * 3 * (rgb_dtype == SAMROAD_U8 ? 1 : 4);
  const size_t sc_bytes = static_cast<size_t>(B) * P * P * 2 * 4;
  const size_t em_bytes = static_cast<size_t>(B) * 256 * s * s * 4;
  const bool topo = points_host && pairs_host && valid_host && Ns > 0 && N > 0;
  const size_t pt_sz = pts_dtype == SAMROAD_I64 ? 8 : 4, pr_sz = pairs_dtype == SAMROAD_I64 ? 8 : 4;
  const size_t pts_bytes = topo ? static_cast<size_t>(B) * N * 2 * pt_sz : 0;
  const size_t prs_bytes = topo ? static_cast<size_t>(B) * Ns * Np * 2 * pr_sz : 0;
  const size_t val_bytes = topo ? static_cast<size_t>(B) * Ns * Np : 0;
  const size_t ts_bytes = topo ? static_cast<size_t>(B) * Ns * Np * 4 : 0;
  // the slot's input staging: tiles, then TopoNet's points, pairs and valid flags, then the topology scores
  struct Staging { char *rgb, *pts, *prs, *val, *ts; size_t bytes; };
  auto staging = [&](void* at) {
    Layout L(at);
    Staging g;
    g.rgb = L.take<char>(in_bytes);
    g.pts = L.take<char>(pts_bytes);
    g.prs = L.take<char>(prs_bytes);
    g.val = L.take<char>(val_bytes);
    g.ts = L.take<char>(ts_bytes);
    g.bytes = L.bytes();
    return g;
  };
  samroad_ctx::HostSlot& sl = h->slots[slot];
  if (!h->s_compute) {
    SRB_CUDA_OK(cudaStreamCreateWithFlags(&h->s_h2d, cudaStreamNonBlocking));
    SRB_CUDA_OK(cudaStreamCreateWithFlags(&h->s_compute, cudaStreamNonBlocking));
    SRB_CUDA_OK(cudaStreamCreateWithFlags(&h->s_copy, cudaStreamNonBlocking));
  }
  if (!sl.ev_done) {
    for (cudaEvent_t* e : {&sl.ev_h2d, &sl.ev_emb, &sl.ev_scores, &sl.ev_compute, &sl.ev_done})
      SRB_CUDA_OK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  }
  const char* what = "samroad_infer_batch_host_async";
  SRB_TRY(grow(sl.in, staging(nullptr).bytes, what));
  SRB_TRY(grow(sl.scores, sc_bytes, what));
  SRB_TRY(grow(sl.emb, em_bytes, what));
  // the activation workspace is shared by both slots: grow it before anything is in flight on it
  SRB_TRY(grow(h->ws, layout_enc(h, B, nullptr).total, what));
  if (topo) SRB_TRY(grow(h->topo_ws, layout_topo(B, N, Ns, Np, nullptr).total, what));
  const Staging io = staging(sl.in.get());
  float* scores = sl.scores.as<float>();
  float* emb = sl.emb.as<float>();
  cudaStream_t su = h->s_h2d, st = h->s_compute, sc = h->s_copy;
  // upload: the slot's input staging was last read by the slot's previous compute
  SRB_CUDA_OK(cudaStreamWaitEvent(su, sl.ev_compute, 0));
  SRB_CUDA_OK(cudaMemcpyAsync(io.rgb, rgb_host, in_bytes, cudaMemcpyHostToDevice, su));
  if (topo) {
    SRB_CUDA_OK(cudaMemcpyAsync(io.pts, points_host, pts_bytes, cudaMemcpyHostToDevice, su));
    SRB_CUDA_OK(cudaMemcpyAsync(io.prs, pairs_host, prs_bytes, cudaMemcpyHostToDevice, su));
    SRB_CUDA_OK(cudaMemcpyAsync(io.val, valid_host, val_bytes, cudaMemcpyHostToDevice, su));
  }
  SRB_CUDA_OK(cudaEventRecord(sl.ev_h2d, su));
  // compute: after the upload, and after the slot's previous results have left its output staging
  SRB_CUDA_OK(cudaStreamWaitEvent(st, sl.ev_h2d, 0));
  SRB_CUDA_OK(cudaStreamWaitEvent(st, sl.ev_done, 0));
  h->ev_emb_hook = sl.ev_emb;
  const int rc_enc = samroad_encode_masks(h, io.rgb, rgb_dtype, B, mask_scores_host ? scores : nullptr,
                                          nullptr, emb, st);
  h->ev_emb_hook = nullptr;
  if (rc_enc != 0) return rc_enc;
  if (image_embeddings_host) {      // the embeddings go back while the mask decoder runs
    SRB_CUDA_OK(cudaStreamWaitEvent(sc, sl.ev_emb, 0));
    SRB_CUDA_OK(cudaMemcpyAsync(image_embeddings_host, emb, em_bytes, cudaMemcpyDeviceToHost, sc));
  }
  if (mask_scores_host) {           // the mask scores while TopoNet runs
    SRB_CUDA_OK(cudaEventRecord(sl.ev_scores, st));
    SRB_CUDA_OK(cudaStreamWaitEvent(sc, sl.ev_scores, 0));
    SRB_CUDA_OK(cudaMemcpyAsync(mask_scores_host, scores, sc_bytes, cudaMemcpyDeviceToHost, sc));
  }
  if (topo)
    SRB_TRY(samroad_toponet(h, emb, io.pts, pts_dtype, io.prs, pairs_dtype,
                            reinterpret_cast<const uint8_t*>(io.val), B, N, Ns, Np, nullptr,
                            reinterpret_cast<float*>(io.ts), st));
  SRB_CUDA_OK(cudaEventRecord(sl.ev_compute, st));
  SRB_CUDA_OK(cudaStreamWaitEvent(sc, sl.ev_compute, 0));
  if (topo && topo_scores_host)
    SRB_CUDA_OK(cudaMemcpyAsync(topo_scores_host, io.ts, ts_bytes, cudaMemcpyDeviceToHost, sc));
  SRB_CUDA_OK(cudaEventRecord(sl.ev_done, sc));
  return 0;
}

// Blocks until everything samroad_infer_batch_host_async queued on `slot` has landed in host memory.
extern "C" int samroad_infer_batch_host_wait(samroad_handle_t h, int slot) {
  SRB_TRY(check_handle(h, true));
  SRB_REQUIRE(slot == 0 || slot == 1, "samroad_infer_batch_host_wait: slot %d (want 0 or 1)", slot);
  if (h->slots[slot].ev_done) SRB_CUDA_OK(cudaEventSynchronize(h->slots[slot].ev_done));
  return 0;
}

// The synchronous form: one batch on slot 0, results in host memory on return.
extern "C" int samroad_infer_batch_host(samroad_handle_t h, const void* rgb_host, int rgb_dtype,
                                        int B, const void* points_host, int pts_dtype,
                                        const void* pairs_host, int pairs_dtype,
                                        const uint8_t* valid_host, int N, int Ns, int Np,
                                        float* mask_scores_host, float* image_embeddings_host,
                                        float* topo_scores_host) {
  SRB_TRY(samroad_infer_batch_host_async(h, 0, rgb_host, rgb_dtype, B, points_host, pts_dtype, pairs_host,
                                         pairs_dtype, valid_host, N, Ns, Np, mask_scores_host,
                                         image_embeddings_host, topo_scores_host));
  return samroad_infer_batch_host_wait(h, 0);
}

extern "C" int samroad_stream_write_value32(void* addr, uint32_t value, void* stream) {
  return stream_write_value32(addr, value, static_cast<cudaStream_t>(stream));
}
extern "C" int samroad_stream_wait_value32(void* addr, uint32_t value, void* stream) {
  return stream_wait_value32_geq(addr, value, static_cast<cudaStream_t>(stream));
}
extern "C" uint64_t samroad_launch_count(int reset) { return launch_count(reset != 0); }
extern "C" const char* samroad_last_error(void) { return get_last_error(); }
extern "C" int samroad_abi_version(void) { return SAMROAD_ABI_VERSION; }

extern "C" int samroad_op_gemm_f16(const void* A, int lda, const void* W, int ldw, int M, int N,
                                   int K, const float* bias, int act, void* out16, int ldo,
                                   void* stream) {
  return gemm_f16out(static_cast<const __half*>(A), lda, static_cast<const __half*>(W), ldw, M, N, K,
                     bias, act, static_cast<__half*>(out16), ldo, static_cast<cudaStream_t>(stream));
}
extern "C" int samroad_op_gemm_f32(const void* A, int lda, const void* W, int ldw, int M, int N,
                                   int K, const float* bias, const float* resid, const float* pos,
                                   int pos_rows, float* out32, int ldo, void* stream) {
  return gemm_f32out(static_cast<const __half*>(A), lda, static_cast<const __half*>(W), ldw, M, N, K,
                     bias, resid, pos, pos_rows, out32, ldo, static_cast<cudaStream_t>(stream));
}
extern "C" int samroad_op_gemm_ln(const void* A, int lda, const void* W, int ldw, int M, int N,
                                  int K, const float* bias, const float* resid, const float* gamma,
                                  const float* beta, float eps, int group, int act, void* out16,
                                  float* out32, float* out_nchw, int tokens, int ldo, void* stream) {
  return gemm_ln(static_cast<const __half*>(A), lda, static_cast<const __half*>(W), ldw, M, N, K,
                 bias, resid, gamma, beta, eps, group, act, static_cast<__half*>(out16), out32,
                 out_nchw, tokens, ldo, static_cast<cudaStream_t>(stream));
}
extern "C" int samroad_op_gemm_ref(const void* A, int lda, const void* W, int ldw, int M, int N,
                                   int K, float* out32, int ldo, void* stream) {
  return gemm_ref_simt(static_cast<const __half*>(A), lda, static_cast<const __half*>(W), ldw, M, N,
                       K, out32, ldo, static_cast<cudaStream_t>(stream));
}
extern "C" int samroad_op_layernorm(const float* x, const float* gamma, const float* beta,
                                    float eps, int M, int D, void* out16, void* stream) {
  return layernorm_f16(x, gamma, beta, eps, M, D, static_cast<__half*>(out16), false,
                       static_cast<cudaStream_t>(stream));
}
extern "C" int samroad_op_attention(const void* qkv16, const float* qkv_bias, const float* rel_h,
                                    const float* rel_w, int B, int s, int win, int heads,
                                    int head_dim, void* out16, void* stream) {
  return encoder_attention(static_cast<const __half*>(qkv16), qkv_bias, rel_h, rel_w, B, s,
                           win, heads, head_dim, static_cast<__half*>(out16),
                           static_cast<cudaStream_t>(stream));
}
extern "C" int samroad_op_sam_decoder(samroad_handle_t h, const float* emb_nchw, int B, float* queries,
                                      float* keys, float* hyper, float* lowres, float* mask_scores,
                                      float* mask_logits, void* stream) {
  SRB_TRY(check_handle(h, false));
  SRB_REQUIRE(h->cfg.use_sam_decoder, "samroad_op_sam_decoder: the handle has no SAM mask decoder");
  SRB_TRY(check_handle(h, true));
  SRB_REQUIRE(emb_nchw, "samroad_op_sam_decoder: null emb_nchw");
  SRB_REQUIRE(B > 0, "samroad_op_sam_decoder: B=%d (want > 0)", B);
  SRB_REQUIRE(mask_scores || mask_logits, "samroad_op_sam_decoder: mask_scores and mask_logits are both null");
  SRB_REQUIRE(static_cast<long>(B) * h->T * 16 < 2147483647L, "batch of %d tiles is too large for one call", B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SRB_TRY(grow(h->sam_ws, sam_decoder_ws_bytes(B, h->T), "samroad_op_sam_decoder"));
  SRB_TRY(sam_decoder_forward(h->sam, emb_nchw, B, h->s, h->cfg.patch_size, h->sam_ws.get(), mask_scores,
                              mask_logits, st));
  return sam_decoder_checkpoints(B, h->T, h->sam_ws.get(), queries, keys, hyper, lowres, st);
}
extern "C" int samroad_op_encoder_taps(samroad_handle_t h, const void* rgb, int rgb_dtype, int B,
                                       const SamroadEncoderTaps* taps, float* mask_scores, float* mask_logits,
                                       float* image_embeddings, void* stream) {
  SRB_TRY(check_handle(h, false));
  if (taps) {
    const int depth = h->cfg.depth;
    SRB_REQUIRE(depth >= 64 || (taps->block_mask >> depth) == 0,
                "samroad_op_encoder_taps: block_mask 0x%llx selects a block >= depth %d",
                static_cast<unsigned long long>(taps->block_mask), depth);
    SRB_REQUIRE(taps->detail_block >= -1 && taps->detail_block < depth,
                "samroad_op_encoder_taps: detail_block=%d (want -1 or a block < depth %d)", taps->detail_block,
                depth);
  }
  h->taps = taps;
  const int rc = samroad_encode_masks(h, rgb, rgb_dtype, B, mask_scores, mask_logits, image_embeddings, stream);
  h->taps = nullptr;
  return rc;
}
extern "C" void samroad_debug_force_simt_attention(int on) { attention_force_simt(on); }
extern "C" int samroad_debug_attention_path(int s, int win, int head_dim, int* q_stages, int* kv_stages) {
  return attention_path(s, win, head_dim, q_stages, kv_stages);
}
extern "C" void samroad_debug_disable_2cta_gemm(int off) { g_ln_ascending = (off & 16) != 0; }
