// sam_road_b200 :: internal C++ launcher declarations (host side).  Every launcher is stream-ordered,
// asynchronous, returns 0 on success and sets srb::set_last_error() otherwise.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace srb {

enum Act : int { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2 };

void set_last_error(const char* fmt, ...);
const char* get_last_error();
int device_sm_count();
// true the first time it is called with this mask on the current CUDA device (then sets the bit)
bool first_use_on_device(uint64_t* device_mask);
void note_launch(int n = 1);
// stream memory operations on a 32-bit flag word (no kernel): ordered write / wait until *addr >= value
int stream_write_value32(void* addr, uint32_t value, cudaStream_t st);
int stream_wait_value32_geq(void* addr, uint32_t value, cudaStream_t st);
uint64_t launch_count(bool reset);

// ---- GEMM family (gemm_ops.cu) : C = A[M,K] * W[N,K]^T with fused epilogues ------------------------
int gemm_f16out(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                const float* bias, int act, __half* out, int ldo, cudaStream_t st);
int gemm_f32out(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                const float* bias, const float* resid, const float* pos, int pos_rows, float* out,
                int ldo, cudaStream_t st);
int gemm_ln(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
            const float* bias, const float* resid, const float* gamma, const float* beta, float eps,
            int group, int act, __half* out16, float* out32, float* out_nchw, int tokens, int ldo,
            cudaStream_t st, int conv_s = 0);   // conv_s > 0: A is an NHWC image, implicit 3x3 / pad 1 conv
int gemm_dec_final(const __half* A, int lda, const __half* W, int ldw, int M, int K,
                   const float* bias3, const float* w4, const float* bias4, int s, int P,
                   float* scores, float* logits, cudaStream_t st);
// plain SIMT fp32-accumulate GEMM used only by the on-device unit tests as an independent checker
int gemm_ref_simt(const __half* A, int lda, const __half* W, int ldw, int M, int N, int K,
                  float* out, int ldo, cudaStream_t st);

// ---- elementwise / data-movement kernels (kernels.cu) ------------------------------------------------
// reverse: walk the rows from the last to the first
int layernorm_f16(const float* x, const float* gamma, const float* beta, float eps, int M, int D,
                  __half* out, bool reverse, cudaStream_t st);
// rgb: [B,P,P,3] fp32 (dtype 0) or uint8 (dtype 1); out: [B*(P/16)^2, 768] fp16, k = ky*48+kx*3+c
int im2col_patch16(const void* rgb, int dtype, int B, int P, const float* mean, const float* inv_std,
                   __half* out, cudaStream_t st);
// scene: uint8 [H,W,3]; tile_xy: device int32 [B,2] origins (x0,y0) inside the scene; out: uint8 [B,P,P,3]
int crop_tiles(const uint8_t* scene, int H, int W, const int* tile_xy, int B, int P, uint8_t* out,
               cudaStream_t st);
// x: [B*s*s, C] fp16 NHWC; out: [B*s*s, 9*C], k = (ky*3+kx)*C + c, zero padding 1
int im2col_3x3(const __half* x, int B, int s, int C, __half* out, cudaStream_t st);
int convert_f32_f16(const float* x, long n, __half* out, cudaStream_t st);

// ---- encoder attention (attention.cu) --------------------------------------------------------------------
// qkv: [B*s*s, 3*D] fp16, columns (q|k|v) x head x hd ; out: [B*s*s, D] fp16.
// win == s means global attention; otherwise window attention over zero-padded LN output, whose pad
// tokens have q=k=v=bias (image_encoder.py:168-172,227); win > s is a single padded window.
// rel_h/rel_w: [2*win-1, hd] fp32.
int encoder_attention(const __half* qkv, const float* qkv_bias, const float* rel_h,
                      const float* rel_w, int B, int s, int win, int heads, int hd, __half* out,
                      cudaStream_t st);
// force the SIMT attention kernel (tests use it as the independent on-device checker)
void attention_force_simt(int mode);   // bit 0: SIMT kernel

// ---- TopoNet pieces (toponet.cu) -----------------------------------------------------------------------------
// points dtype: 0 = float32, 1 = int64, 2 = int32 ; pairs dtype: 1 = int64, 2 = int32
int topo_sample_features(const float* feat_nchw, int B, int C, int s, int P, const void* points,
                         int pts_dtype, int N, __half* out, cudaStream_t st);
int topo_sample_features_f32(const float* feat_nchw, int B, int C, int s, int P, const void* points,
                             int pts_dtype, int N, float* out, cudaStream_t st);
// pair features (model.py:96-120): x = relu(Ws f[src] + Wt f[tgt] + Wo (pt[tgt] - pt[src]) + bias)
struct TopoPairInputs {
  const float* pst;          // [B*N, 256] per-point projections (Ws f | Wt f)
  const float* w_off;        // [128][2]
  const float* bias;         // [128]
  const void* points;        // [B, N, 2]
  const void* pairs;         // [B, Ns, Np, 2]
  int pts_dtype, pairs_dtype, N, tokens_per_b, zero_offset;
};
int topo_pair_features(const TopoPairInputs& in, int tokens, float* x32, __half* x16, cudaStream_t st);
int topo_fix_valid(const uint8_t* valid, int rows, int Np, uint8_t* out, cudaStream_t st);
int topo_attention(const __half* qkv, const uint8_t* valid, int rows, int Np, __half* out,
                   cudaStream_t st);
int topo_output(const float* x32, const uint8_t* valid_fixed, const float* w, const float* b,
                int tokens, float* logits, float* scores, cudaStream_t st);

// fp32 parameters of one post-norm encoder layer (torch TransformerEncoderLayer, d = 128)
struct TopoLayerParams {
  const float* in_b;    // [384]
  const float* out_b;   // [128]
  const float* l1_b;    // [128]
  const float* l2_b;    // [128]
  const float *n1_g, *n1_b, *n2_g, *n2_b;   // [128]
};
// fused 3-layer transformer + output_proj for n_pairs Np == 16 or 32 (toponet_tc.cuh).  w_chunks: per
// layer Wq, Wk, Wv, Wo, W1, W2 as [128, 128] fp16 blocks; out_w [128], out_b [1].
int topo_transformer_fused(const TopoPairInputs& in, const __half* w_chunks, const TopoLayerParams* layers,
                           const float* out_w, const float* out_b, const uint8_t* valid_fixed, int tokens,
                           int Np, float* logits, float* scores, cudaStream_t st);

// ---- SAM mask-decoder path (sam_decoder.cu), USE_SAM_DECODER: True --------------------------------
struct SamAttnW { const float *qw, *qb, *kw, *kb, *vw, *vb, *ow, *ob; };
struct SamDecoderWeights {
  const float* tokens;        // [4][256] = [iou_token ; mask_tokens]
  const float* q0;            // [4][256] = norm1(self_attn(tokens)) of layer 0 (sam_decoder_prepare)
  const float* no_mask_embed; // [256]
  const float* dense_pe;      // [T][256]
  SamAttnW self_attn[2], t2i[2], i2t[2], final_attn;
  const float *n1g[2], *n1b[2], *n2g[2], *n2b[2], *n3g[2], *n3b[2], *n4g[2], *n4b[2];
  const float *l1w[2], *l1b[2], *l2w[2], *l2b[2];
  const float *nfg, *nfb;
  const float* hw[2][3];      // hypernetwork MLPs 1 and 2
  const float* hb[2][3];
  const __half *t2i_kw16[3], *t2i_vw16[3];   // image-side GEMM operands (layers 0, 1, final)
  const __half *i2t_qw16[2], *i2t_ow16[2];
  const __half *up1_w, *up2_w;
  const float *up1_b, *up1_g, *up1_beta, *up2_b;
};
size_t sam_decoder_ws_bytes(int B, int T);
int sam_decoder_prepare(const SamDecoderWeights& w, float* q0_out, cudaStream_t st);
int sam_decoder_forward(const SamDecoderWeights& w, const float* emb_nchw, int B, int s, int P, void* ws,
                        float* mask_scores, float* mask_logits, cudaStream_t st);

// ---- mask fusion (kernels.cu) : inferencer.py:79-110 --------------------------------------------------------
int fuse_masks(const float* scores, int n_tiles, int P, const int* tile_x0, const int* tile_y0,
               int H, int W, uint8_t* keypoint_u8, uint8_t* road_u8, cudaStream_t st);

}  // namespace srb
