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

// ---- staged-tensor access -----------------------------------------------------------------------
struct Packer {
  samroad_ctx* h;
  bool ok = true;
  char msg[512] = "";

  const HostTensor* get(const std::string& key, std::initializer_list<int64_t> shape) {
    auto it = h->staged.find(key);
    if (it == h->staged.end()) {
      fail("missing state_dict key '%s'", key.c_str());
      return nullptr;
    }
    const HostTensor& t = it->second;
    bool same = t.shape.size() == shape.size();
    if (same) {
      size_t i = 0;
      for (auto d : shape) same = same && (t.shape[i++] == d);
    }
    if (!same) {
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
  template <typename T>
  T* upload(const std::vector<T>& v) {
    if (!ok) return nullptr;
    DeviceBuffer d;
    if (d.reserve(v.size() * sizeof(T) + 256, "samroad_finalize_weights")) {
      fail("cudaMalloc of %zu bytes for weights failed", v.size() * sizeof(T));
      return nullptr;
    }
    T* p = d.as<T>();
    h->weight_allocs.push_back(std::move(d));
    if (cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) {
      fail("cudaMemcpy of weights failed");
      return nullptr;
    }
    return p;
  }
  float* f32(const std::string& key, std::initializer_list<int64_t> shape) {
    const HostTensor* t = get(key, shape);
    return t ? upload(t->data) : nullptr;
  }
  static std::vector<__half> to_half(const std::vector<float>& v) {
    std::vector<__half> o(v.size());
    for (size_t i = 0; i < v.size(); ++i) o[i] = __float2half_rn(v[i]);
    return o;
  }
  // nn.Linear weight [out, in] is already the K-major [N, K] operand
  __half* linear_w(const std::string& key, int64_t n, int64_t k) {
    const HostTensor* t = get(key, {n, k});
    return t ? upload(to_half(t->data)) : nullptr;
  }
};

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

// ConvTranspose2d(k=2,s=2) weight [Cin, Cout, 2, 2] -> GEMM operand [N = (d, co), K = ci] with
// d = di*2 + dj, so that output column block d is sub-pixel (di,dj) (SURVEY.md §8a P7).
std::vector<__half> pack_convT(const HostTensor& w, int cin, int cout) {
  std::vector<__half> o(static_cast<size_t>(4) * cout * cin);
  for (int ci = 0; ci < cin; ++ci)
    for (int co = 0; co < cout; ++co)
      for (int d = 0; d < 4; ++d)
        o[(static_cast<size_t>(d) * cout + co) * cin + ci] =
            __float2half_rn(w.data[(static_cast<size_t>(ci) * cout + co) * 4 + d]);
  return o;
}
std::vector<float> tile4(const std::vector<float>& b) {
  std::vector<float> o(b.size() * 4);
  for (int d = 0; d < 4; ++d)
    for (size_t i = 0; i < b.size(); ++i) o[d * b.size() + i] = b[i];
  return o;
}

// Grows a workspace or staging buffer to `need` bytes.  The handle's three streams may still read the old
// block, so the device is synchronised before it is replaced.
int grow(DeviceBuffer& b, size_t need, const char* what) {
  if (need <= b.capacity()) return 0;
  if (b.get()) SRB_CUDA_OK(cudaDeviceSynchronize());
  return b.reserve(need, what);
}

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
  // drop previously packed weights (re-load after load_state_dict)
  SRB_CUDA_OK(cudaDeviceSynchronize());
  h->weight_allocs.clear();
  h->blocks.clear();

  Packer P{h};
  const SamRoadCfg& c = h->cfg;
  const int64_t D = h->D, s = h->s, hd = h->hd;

  // ---- patch embed: [D,3,16,16] -> [D, 768] with k = ky*48 + kx*3 + c (matches im2col_patch16) ----
  if (const HostTensor* w = P.get("image_encoder.patch_embed.proj.weight", {D, 3, 16, 16})) {
    std::vector<__half> o(static_cast<size_t>(D) * 768);
    for (int64_t n = 0; n < D; ++n)
      for (int ch = 0; ch < 3; ++ch)
        for (int ky = 0; ky < 16; ++ky)
          for (int kx = 0; kx < 16; ++kx)
            o[n * 768 + ky * 48 + kx * 3 + ch] =
                __float2half_rn(w->data[((n * 3 + ch) * 16 + ky) * 16 + kx]);
    h->pe_w = P.upload(o);
  }
  h->pe_b = P.f32("image_encoder.patch_embed.proj.bias", {D});
  h->pos = P.f32("image_encoder.pos_embed", {1, s, s, D});

  // ---- transformer blocks ----
  h->blocks.resize(c.depth);
  for (int i = 0; i < c.depth && P.ok; ++i) {
    BlockW& b = h->blocks[i];
    const bool glob = is_global_block(c, i);
    // A window block keeps its window size even when it exceeds the grid (s < 14, PATCH_SIZE < 224):
    // the s x s tokens are then padded to one window, whose pad tokens are softmax keys
    // (image_encoder.py:168-172), and the rel-pos tables have 2*window-1 rows.
    b.win = glob ? static_cast<int>(s) : c.window_size;
    const int64_t rel_rows = glob ? 2 * s - 1 : 2 * c.window_size - 1;
    auto K = [&](const char* suffix) { return fmt_key("image_encoder.blocks.%d.", i) + suffix; };
    b.ln1_g = P.f32(K("norm1.weight"), {D});
    b.ln1_b = P.f32(K("norm1.bias"), {D});
    b.ln2_g = P.f32(K("norm2.weight"), {D});
    b.ln2_b = P.f32(K("norm2.bias"), {D});
    // qkv (+ LoRA merge: qkv = xW^T + b ; q += B_q A_q x ; v += B_v A_v x   model.py:179-186)
    if (const HostTensor* w = P.get(K("attn.qkv.weight"), {3 * D, D})) {
      std::vector<float> wf = w->data;
      if (c.lora_rank > 0) {
        const int64_t r = c.lora_rank;
        const HostTensor* aq = P.get(K("attn.qkv.linear_a_q.weight"), {r, D});
        const HostTensor* bq = P.get(K("attn.qkv.linear_b_q.weight"), {D, r});
        const HostTensor* av = P.get(K("attn.qkv.linear_a_v.weight"), {r, D});
        const HostTensor* bv = P.get(K("attn.qkv.linear_b_v.weight"), {D, r});
        if (aq && bq && av && bv) {
          for (int64_t n = 0; n < D; ++n)
            for (int64_t j = 0; j < r; ++j) {
              const float bqv = bq->data[n * r + j], bvv = bv->data[n * r + j];
              float* wq = &wf[n * D];
              float* wv = &wf[(2 * D + n) * D];
              const float* aqr = &aq->data[j * D];
              const float* avr = &av->data[j * D];
              for (int64_t k = 0; k < D; ++k) {
                wq[k] += bqv * aqr[k];
                wv[k] += bvv * avr[k];
              }
            }
        }
      }
      b.qkv_w = P.upload(Packer::to_half(wf));
    }
    b.qkv_b = P.f32(K("attn.qkv.bias"), {3 * D});
    b.proj_w = P.linear_w(K("attn.proj.weight"), D, D);
    b.proj_b = P.f32(K("attn.proj.bias"), {D});
    b.rel_h = P.f32(K("attn.rel_pos_h"), {rel_rows, hd});
    b.rel_w = P.f32(K("attn.rel_pos_w"), {rel_rows, hd});
    b.lin1_w = P.linear_w(K("mlp.lin1.weight"), 4 * D, D);
    b.lin1_b = P.f32(K("mlp.lin1.bias"), {4 * D});
    b.lin2_w = P.linear_w(K("mlp.lin2.weight"), D, 4 * D);
    b.lin2_b = P.f32(K("mlp.lin2.bias"), {D});
    if (!glob && c.window_size > 64)
      P.fail("window_size=%d unsupported (at most 64)", c.window_size);
  }

  // ---- neck (image_encoder.py:88-104) ----
  if (const HostTensor* w = P.get("image_encoder.neck.0.weight", {256, D, 1, 1}))
    h->neck0_w = P.upload(Packer::to_half(w->data));
  h->neck1_g = P.f32("image_encoder.neck.1.weight", {256});
  h->neck1_b = P.f32("image_encoder.neck.1.bias", {256});
  if (const HostTensor* w = P.get("image_encoder.neck.2.weight", {256, 256, 3, 3})) {
    std::vector<__half> o(static_cast<size_t>(256) * 2304);   // [n][tap*256 + c]
    for (int n = 0; n < 256; ++n)
      for (int ch = 0; ch < 256; ++ch)
        for (int tap = 0; tap < 9; ++tap)
          o[static_cast<size_t>(n) * 2304 + tap * 256 + ch] =
              __float2half_rn(w->data[(static_cast<size_t>(n) * 256 + ch) * 9 + tap]);
    h->neck2_w = P.upload(o);
  }
  h->neck3_g = P.f32("image_encoder.neck.3.weight", {256});
  h->neck3_b = P.f32("image_encoder.neck.3.bias", {256});

  if (!c.use_sam_decoder) {
  // ---- naive map decoder (model.py:286-295) ----
  if (const HostTensor* w = P.get("map_decoder.0.weight", {256, 128, 2, 2}))
    h->dec1_w = P.upload(pack_convT(*w, 256, 128));
  if (const HostTensor* b = P.get("map_decoder.0.bias", {128})) h->dec1_b = P.upload(tile4(b->data));
  h->dec_ln_g = P.f32("map_decoder.1.weight", {128});
  h->dec_ln_b = P.f32("map_decoder.1.bias", {128});
  if (const HostTensor* w = P.get("map_decoder.3.weight", {128, 64, 2, 2}))
    h->dec2_w = P.upload(pack_convT(*w, 128, 64));
  if (const HostTensor* b = P.get("map_decoder.3.bias", {64})) h->dec2_b = P.upload(tile4(b->data));
  if (const HostTensor* w = P.get("map_decoder.5.weight", {64, 32, 2, 2}))
    h->dec3_w = P.upload(pack_convT(*w, 64, 32));
  h->dec3_b = P.f32("map_decoder.5.bias", {32});
  if (const HostTensor* w = P.get("map_decoder.7.weight", {32, 2, 2, 2})) {
    std::vector<float> o(32 * 8);   // [ci][di*4 + dj*2 + co]
    for (int ci = 0; ci < 32; ++ci)
      for (int co = 0; co < 2; ++co)
        for (int d = 0; d < 4; ++d) o[ci * 8 + d * 2 + co] = w->data[(ci * 2 + co) * 4 + d];
    h->dec4_w = P.upload(o);
  }
  h->dec4_b = P.f32("map_decoder.7.bias", {2});

  } else {
    // ---- SAM mask decoder + null-prompt encoder (model.py:260-282) ----
    SamDecoderWeights& S = h->sam;
    const std::string md = "mask_decoder.", tr = "mask_decoder.transformer.";
    if (const HostTensor* it = P.get(md + "iou_token.weight", {1, 256})) {
      if (const HostTensor* mt = P.get(md + "mask_tokens.weight", {3, 256})) {
        std::vector<float> tok(it->data);
        tok.insert(tok.end(), mt->data.begin(), mt->data.end());
        S.tokens = P.upload(tok);
      }
    }
    S.no_mask_embed = P.f32("prompt_encoder.no_mask_embed.weight", {1, 256});
    if (const HostTensor* G = P.get("prompt_encoder.pe_layer.positional_encoding_gaussian_matrix", {2, 128})) {
      // PromptEncoder.get_dense_pe (prompt_encoder.py:62-71,185-205): constant per config
      std::vector<float> pe(static_cast<size_t>(s) * s * 256);
      for (int y = 0; y < s; ++y)
        for (int x = 0; x < s; ++x) {
          const float cx = 2.0f * ((x + 0.5f) / s) - 1.0f, cy = 2.0f * ((y + 0.5f) / s) - 1.0f;
          for (int k = 0; k < 128; ++k) {
            const float a = 6.283185307179586f * (cx * G->data[k] + cy * G->data[128 + k]);
            pe[(static_cast<size_t>(y) * s + x) * 256 + k] = sinf(a);
            pe[(static_cast<size_t>(y) * s + x) * 256 + 128 + k] = cosf(a);
          }
        }
      S.dense_pe = P.upload(pe);
    }
    auto attn = [&](const std::string& p, int64_t internal) {
      SamAttnW a;
      a.qw = P.f32(p + "q_proj.weight", {internal, 256}); a.qb = P.f32(p + "q_proj.bias", {internal});
      a.kw = P.f32(p + "k_proj.weight", {internal, 256}); a.kb = P.f32(p + "k_proj.bias", {internal});
      a.vw = P.f32(p + "v_proj.weight", {internal, 256}); a.vb = P.f32(p + "v_proj.bias", {internal});
      a.ow = P.f32(p + "out_proj.weight", {256, internal}); a.ob = P.f32(p + "out_proj.bias", {256});
      return a;
    };
    for (int l = 0; l < 2; ++l) {
      const std::string p = tr + "layers." + std::to_string(l) + ".";
      S.self_attn[l] = attn(p + "self_attn.", 256);
      S.t2i[l] = attn(p + "cross_attn_token_to_image.", 128);
      S.i2t[l] = attn(p + "cross_attn_image_to_token.", 128);
      S.n1g[l] = P.f32(p + "norm1.weight", {256}); S.n1b[l] = P.f32(p + "norm1.bias", {256});
      S.n2g[l] = P.f32(p + "norm2.weight", {256}); S.n2b[l] = P.f32(p + "norm2.bias", {256});
      S.n3g[l] = P.f32(p + "norm3.weight", {256}); S.n3b[l] = P.f32(p + "norm3.bias", {256});
      S.n4g[l] = P.f32(p + "norm4.weight", {256}); S.n4b[l] = P.f32(p + "norm4.bias", {256});
      S.l1w[l] = P.f32(p + "mlp.lin1.weight", {2048, 256}); S.l1b[l] = P.f32(p + "mlp.lin1.bias", {2048});
      S.l2w[l] = P.f32(p + "mlp.lin2.weight", {256, 2048}); S.l2b[l] = P.f32(p + "mlp.lin2.bias", {256});
      S.t2i_kw16[l] = P.linear_w(p + "cross_attn_token_to_image.k_proj.weight", 128, 256);
      S.t2i_vw16[l] = P.linear_w(p + "cross_attn_token_to_image.v_proj.weight", 128, 256);
      S.i2t_qw16[l] = P.linear_w(p + "cross_attn_image_to_token.q_proj.weight", 128, 256);
      S.i2t_ow16[l] = P.linear_w(p + "cross_attn_image_to_token.out_proj.weight", 256, 128);
    }
    S.final_attn = attn(tr + "final_attn_token_to_image.", 128);
    S.t2i_kw16[2] = P.linear_w(tr + "final_attn_token_to_image.k_proj.weight", 128, 256);
    S.t2i_vw16[2] = P.linear_w(tr + "final_attn_token_to_image.v_proj.weight", 128, 256);
    S.nfg = P.f32(tr + "norm_final_attn.weight", {256}); S.nfb = P.f32(tr + "norm_final_attn.bias", {256});
    for (int mi = 0; mi < 2; ++mi)
      for (int j = 0; j < 3; ++j) {
        const std::string k = md + "output_hypernetworks_mlps." + std::to_string(mi + 1) + ".layers." +
                              std::to_string(j) + ".";
        const int64_t out = j == 2 ? 32 : 256;
        S.hw[mi][j] = P.f32(k + "weight", {out, 256});
        S.hb[mi][j] = P.f32(k + "bias", {out});
      }
    if (const HostTensor* wt = P.get(md + "output_upscaling.0.weight", {256, 64, 2, 2}))
      S.up1_w = P.upload(pack_convT(*wt, 256, 64));
    if (const HostTensor* bt = P.get(md + "output_upscaling.0.bias", {64})) S.up1_b = P.upload(tile4(bt->data));
    S.up1_g = P.f32(md + "output_upscaling.1.weight", {64});
    S.up1_beta = P.f32(md + "output_upscaling.1.bias", {64});
    if (const HostTensor* wt = P.get(md + "output_upscaling.3.weight", {64, 32, 2, 2}))
      S.up2_w = P.upload(pack_convT(*wt, 64, 32));
    if (const HostTensor* bt = P.get(md + "output_upscaling.3.bias", {32})) S.up2_b = P.upload(tile4(bt->data));
    if (P.ok) {   // constant part of the decoder: layer-0 queries
      float* q0 = P.upload(std::vector<float>(4 * 256, 0.f));
      if (q0 && (sam_decoder_prepare(S, q0, nullptr) != 0 || cudaStreamSynchronize(nullptr) != cudaSuccess))
        P.fail("sam_decoder_prepare failed: %s", get_last_error());
      S.q0 = q0;
    }
  }

  // ---- TopoNet (model.py:61-86) ----
  h->tp_feat_w = P.linear_w("topo_net.feature_proj.weight", 128, 256);
  h->tp_feat_b = P.f32("topo_net.feature_proj.bias", {128});
  if (const HostTensor* w = P.get("topo_net.pair_proj.weight", {128, 258})) {
    std::vector<__half> st(static_cast<size_t>(256) * 128);   // rows 0..127: Ws, 128..255: Wt
    std::vector<float> off(128 * 2);
    for (int n = 0; n < 128; ++n) {
      for (int k = 0; k < 128; ++k) {
        st[static_cast<size_t>(n) * 128 + k] = __float2half_rn(w->data[n * 258 + k]);
        st[static_cast<size_t>(128 + n) * 128 + k] = __float2half_rn(w->data[n * 258 + 128 + k]);
      }
      off[n * 2 + 0] = w->data[n * 258 + 256];
      off[n * 2 + 1] = w->data[n * 258 + 257];
    }
    h->tp_st_w = P.upload(st);
    h->tp_off_w = P.upload(off);
  }
  h->tp_pair_b = P.f32("topo_net.pair_proj.bias", {128});
  if (c.toponet_version != SAMROAD_TOPO_NO_TRANSFORMER) {
    std::vector<__half> chunks(static_cast<size_t>(18) * 128 * 128);
    for (int l = 0; l < 3 && P.ok; ++l) {
      TopoLayerParams& t = h->tp_layers[l];
      auto K = [&](const char* suffix) {
        return fmt_key("topo_net.transformer_encoder.layers.%d.", l) + suffix;
      };
      const HostTensor* src[4] = {P.get(K("self_attn.in_proj_weight"), {384, 128}),
                                  P.get(K("self_attn.out_proj.weight"), {128, 128}),
                                  P.get(K("linear1.weight"), {128, 128}),
                                  P.get(K("linear2.weight"), {128, 128})};
      size_t off = static_cast<size_t>(l) * 6 * 128 * 128;
      for (int i = 0; i < 4 && P.ok; ++i) {
        for (size_t j = 0; j < src[i]->data.size(); ++j) chunks[off + j] = __float2half_rn(src[i]->data[j]);
        off += src[i]->data.size();
      }
      t.in_b = P.f32(K("self_attn.in_proj_bias"), {384});
      t.out_b = P.f32(K("self_attn.out_proj.bias"), {128});
      t.l1_b = P.f32(K("linear1.bias"), {128});
      t.l2_b = P.f32(K("linear2.bias"), {128});
      t.n1_g = P.f32(K("norm1.weight"), {128});
      t.n1_b = P.f32(K("norm1.bias"), {128});
      t.n2_g = P.f32(K("norm2.weight"), {128});
      t.n2_b = P.f32(K("norm2.bias"), {128});
    }
    h->tp_chunks = P.upload(chunks);
  }
  h->tp_out_w = P.f32("topo_net.output_proj.weight", {1, 128});
  h->tp_out_b = P.f32("topo_net.output_proj.bias", {1});

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

// ---- device repack of one head tensor (samroad_update_tensor_device) ------------------------------------------
namespace {

enum RepackMode { RP_COPY, RP_CONVT, RP_TILE4, RP_DEC4, RP_PAIR_ST, RP_PAIR_OFF };

// dst[i] = src[index(i)] for the packings of samroad_finalize_weights, fp16 (round to nearest even, as the host
// pack) or fp32
__global__ void repack_kernel(const float* __restrict__ src, int mode, int cin, int cout, long long n, float* d32,
                              __half* d16) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long j = i;
  switch (mode) {
    case RP_CONVT: {   // o[(d*cout + co)*cin + ci] = w[(ci*cout + co)*4 + d]
      const long long ci = i % cin, dc = i / cin, co = dc % cout, d = dc / cout;
      j = (ci * cout + co) * 4 + d;
      break;
    }
    case RP_TILE4: j = i % cout; break;
    case RP_DEC4: {    // o[ci*8 + d*2 + co] = w[(ci*2 + co)*4 + d]
      const long long ci = i / 8, d = (i % 8) / 2, co = i % 2;
      j = (ci * 2 + co) * 4 + d;
      break;
    }
    case RP_PAIR_ST: {   // rows 0..127: Ws, 128..255: Wt of pair_proj.weight [128, 258]
      const long long r = i / 128, k = i % 128;
      j = (r % 128) * 258 + (r / 128) * 128 + k;
      break;
    }
    case RP_PAIR_OFF: j = (i / 2) * 258 + 256 + i % 2; break;
    default: break;
  }
  const float v = src[j];
  if (d16) d16[i] = __float2half_rn(v);
  else d32[i] = v;
}

}  // namespace

extern "C" int samroad_update_tensor_device(samroad_handle_t h, const char* key, const float* dev_data,
                                            const int64_t* shape, int ndim, void* stream) {
  SRB_TRY(check_handle(h, true));
  SRB_REQUIRE(key && dev_data && (shape || ndim == 0) && ndim >= 0 && ndim <= 8,
              "samroad_update_tensor_device: bad arguments");
  SRB_REQUIRE(!h->cfg.use_sam_decoder, "samroad_update_tensor_device: the SAM mask decoder is repacked on the host only");
  const std::string k = key;
  struct Target { int mode; int cin, cout; long long n; float* d32; __half* d16; };
  std::vector<Target> tg;
  std::vector<int64_t> want;
  auto f32 = [&](const float* p, long long n) { tg.push_back({RP_COPY, 0, 0, n, const_cast<float*>(p), nullptr}); };
  auto f16 = [&](const __half* p, long long n) { tg.push_back({RP_COPY, 0, 0, n, nullptr, const_cast<__half*>(p)}); };
  if (k == "map_decoder.0.weight") { want = {256, 128, 2, 2}; tg.push_back({RP_CONVT, 256, 128, 4LL * 128 * 256, nullptr, h->dec1_w}); }
  else if (k == "map_decoder.0.bias") { want = {128}; tg.push_back({RP_TILE4, 0, 128, 512, h->dec1_b, nullptr}); }
  else if (k == "map_decoder.1.weight") { want = {128}; f32(h->dec_ln_g, 128); }
  else if (k == "map_decoder.1.bias") { want = {128}; f32(h->dec_ln_b, 128); }
  else if (k == "map_decoder.3.weight") { want = {128, 64, 2, 2}; tg.push_back({RP_CONVT, 128, 64, 4LL * 64 * 128, nullptr, h->dec2_w}); }
  else if (k == "map_decoder.3.bias") { want = {64}; tg.push_back({RP_TILE4, 0, 64, 256, h->dec2_b, nullptr}); }
  else if (k == "map_decoder.5.weight") { want = {64, 32, 2, 2}; tg.push_back({RP_CONVT, 64, 32, 4LL * 32 * 64, nullptr, h->dec3_w}); }
  else if (k == "map_decoder.5.bias") { want = {32}; f32(h->dec3_b, 32); }
  else if (k == "map_decoder.7.weight") { want = {32, 2, 2, 2}; tg.push_back({RP_DEC4, 0, 0, 256, h->dec4_w, nullptr}); }
  else if (k == "map_decoder.7.bias") { want = {2}; f32(h->dec4_b, 2); }
  else if (k == "topo_net.feature_proj.weight") { want = {128, 256}; f16(h->tp_feat_w, 128 * 256); }
  else if (k == "topo_net.feature_proj.bias") { want = {128}; f32(h->tp_feat_b, 128); }
  else if (k == "topo_net.pair_proj.weight") {
    want = {128, 258};
    tg.push_back({RP_PAIR_ST, 0, 0, 256 * 128, nullptr, h->tp_st_w});
    tg.push_back({RP_PAIR_OFF, 0, 0, 256, h->tp_off_w, nullptr});
  }
  else if (k == "topo_net.pair_proj.bias") { want = {128}; f32(h->tp_pair_b, 128); }
  else if (k == "topo_net.output_proj.weight") { want = {1, 128}; f32(h->tp_out_w, 128); }
  else if (k == "topo_net.output_proj.bias") { want = {1}; f32(h->tp_out_b, 1); }
  else if (h->cfg.toponet_version != SAMROAD_TOPO_NO_TRANSFORMER &&
           k.rfind("topo_net.transformer_encoder.layers.", 0) == 0 && k.size() > 38 && k[37] == '.' &&
           k[36] >= '0' && k[36] <= '2') {
    const int l = k[36] - '0';
    const std::string s = k.substr(38);
    const TopoLayerParams& t = h->tp_layers[l];
    const __half* chunk = h->tp_chunks + static_cast<size_t>(l) * 6 * 128 * 128;
    if (s == "self_attn.in_proj_weight") { want = {384, 128}; f16(chunk, 384 * 128); }
    else if (s == "self_attn.out_proj.weight") { want = {128, 128}; f16(chunk + 3 * 128 * 128, 128 * 128); }
    else if (s == "linear1.weight") { want = {128, 128}; f16(chunk + 4 * 128 * 128, 128 * 128); }
    else if (s == "linear2.weight") { want = {128, 128}; f16(chunk + 5 * 128 * 128, 128 * 128); }
    else if (s == "self_attn.in_proj_bias") { want = {384}; f32(t.in_b, 384); }
    else if (s == "self_attn.out_proj.bias") { want = {128}; f32(t.out_b, 128); }
    else if (s == "linear1.bias") { want = {128}; f32(t.l1_b, 128); }
    else if (s == "linear2.bias") { want = {128}; f32(t.l2_b, 128); }
    else if (s == "norm1.weight") { want = {128}; f32(t.n1_g, 128); }
    else if (s == "norm1.bias") { want = {128}; f32(t.n1_b, 128); }
    else if (s == "norm2.weight") { want = {128}; f32(t.n2_g, 128); }
    else if (s == "norm2.bias") { want = {128}; f32(t.n2_b, 128); }
  }
  SRB_REQUIRE(!tg.empty(), "samroad_update_tensor_device: '%s' is not a head tensor of this configuration", key);
  bool same = static_cast<size_t>(ndim) == want.size();
  for (int i = 0; same && i < ndim; ++i) same = shape[i] == want[i];
  SRB_REQUIRE(same, "samroad_update_tensor_device: '%s' has the wrong shape", key);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (const Target& t : tg) {
    SRB_LAUNCH(repack_kernel, static_cast<unsigned>((t.n + 255) / 256), 256, 0, st, dev_data, t.mode, t.cin, t.cout,
               t.n, t.d32, t.d16);
  }
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
