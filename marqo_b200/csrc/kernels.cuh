// Memory-bound helper kernels of the encoders (LayerNorm, embeddings, im2col, pooling + projection + L2 normalise,
// dtype conversion).  All are coalesced / vectorised; none is GEMM-shaped.  The wrappers the encoders' forward passes
// call return the number of kernels they launched (0 for an empty batch), which b200_model_last_timing reports.
#pragma once
#include "common.cuh"

namespace mb {
namespace kernels {

// y = LayerNorm(x) * gamma + beta over rows of width w (w % 128 == 0, w <= 1664).  Row r is read at
// x + r * in_stride (floats).  Writes fp32 (out_f32, may alias x) and/or bf16 (out_bf16), both compact [rows, w].
int layernorm(const float* x, long long in_stride, const float* gamma, const float* beta, float eps, int rows, int w,
              float* out_f32, __nv_bfloat16* out_bf16, cudaStream_t s);
// The same over bf16 rows (widened exactly to fp32), bf16 out [rows, w]: EVA02's LayerNorm of the attention output.
int layernorm_bf16(const __nv_bfloat16* x, long long in_stride, const float* gamma, const float* beta, float eps,
                   int rows, int w, __nv_bfloat16* out, cudaStream_t s);

// Rotary position embedding, in place on qkv bf16 [n * S, 3w] (q | k | v, heads of 64): rows first .. S - 1 of each
// sequence (first 1: EVA02, whose class row is not rotated; 0: GTE) are rotated, row s by table row s - first (fp32
// (cos, sin) pairs [S - first, 32]).  Pair j of every q and k head, columns (a, b), becomes (a cos - b sin, b cos + a sin)
// with (cos, sin) = table[(s - first) * 32 + j], computed in fp32 and rounded once.  The columns of pair j are 2j and
// 2j + 1 (INTERLEAVED: EVA02, timm's apply_rot_embed_cat) or j and j + 32 (HALF: NewModel's rotate_half).  The first
// rows and the v columns are left untouched.  w % 64 == 0.
enum class RopePairing { INTERLEAVED, HALF };
int rope_qk(__nv_bfloat16* qkv, int n, int S, int first, int w, const float* table, RopePairing pairing, cudaStream_t s);
// rope_qk's table for a G x G patch grid and timm's ref_feat_shape (ref, ref), on the host, computed in fp64:
// out[(p * 32 + i) * 2 + {0, 1}] = (cos, sin) of pair i of patch p (b200_model_desc: eva_rope_ref_grid).
void rope_table(int G, int ref, float* out);
// rope_qk's table for GTE's 1-D positions 0 .. ctx - 1 (NewModel's NTKScalingRotaryEmbedding, heads of 64, verify), on
// the host, in fp64: out[(s * 32 + j) * 2 + {0, 1}] = (cos, sin) of s f_j with
// f_j = (base factor)^(-2j / 64) / factor^(2 / 64) (b200_model_desc: rope_theta, rope_ntk_factor).
void rope_table_ntk(int ctx, double base, double factor, float* out);

// GeGLU: in bf16 [rows, 2h] holds up (columns 0 .. h - 1) and gate (h .. 2h - 1); out bf16 [rows, h] at row stride ldo
// = GELU_erf(gate) * up, computed in fp32 and rounded once.  out may be the up half of in (ldo = 2h).  h % 8 == 0.
int geglu(const __nv_bfloat16* in, int rows, int h, __nv_bfloat16* out, long long ldo, cudaStream_t s);

// EVA02 SwiGLU + its LayerNorm: in bf16 [rows, 2 hp] holds the gate g (columns 0 .. hp - 1) and x (hp .. 2hp - 1);
// u = SiLU(g) x in fp32, LayerNorm over the h true columns (mean, then variance about it), * gamma + beta [h] -> bf16
// out [rows, hp] at row stride ldo, the pad columns h .. hp - 1 exactly 0.  hp is h rounded up to 64, <= SWIGLU_MAX_HP.
// out may be in itself (ldo = 2 hp): a row is read whole before it is written.
constexpr int SWIGLU_MAX_HP = 3072;
int swiglu_ln(const __nv_bfloat16* in, int rows, int hp, int h, const float* gamma, const float* beta, float eps,
              __nv_bfloat16* out, long long ldo, cudaStream_t s);

// Already-normalised fp32 CHW [n, 3, S, S] -> bf16 A matrix of the ViT token rows [n * (g*g + cls), kpad]: row
// b * (g*g + cls) + t is zero for the class token t < cls (cls is 1 for CLIP, 0 for SigLIP), else patch t - cls
// (row-major in the g x g grid) with k = c*p*p + dy*p + dx, zero for k >= 3*p*p.
int im2col_f32(const float* chw, int n, int S, int p, int kpad, int cls, __nv_bfloat16* out, cudaStream_t s);

// x[b * tokens_per_image + t, :] = positional_embedding[t], plus class_embedding for t == 0 unless cls is NULL
// (w % 4 == 0): the rows the patch-embed GEMM then adds conv1(patch) onto in place
int vit_embed_rows(float* x, const float* cls, const float* pos, int n, int tokens_per_image, int w, cudaStream_t s);

// CLIP text: x[b, s, :] = token_embedding[ids[b, s]] + positional_embedding[s]; also eot[b] = arg-max_s ids[b, s]
int clip_text_embed(const int32_t* ids, const float* tok, const float* pos, int n, int S, int w, int vocab, float* x,
                    int32_t* eot, cudaStream_t s);

// BERT: x = LN(word[ids] + position[s] + token_type[0]); pos NULL (GTE) adds no position row.  fp32 + bf16 copies.  Also kv_len[b] = sum(mask[b, :])
// (mask may be NULL = all ones).
int bert_embed_ln(const int32_t* ids, const int32_t* mask, const float* word, const float* pos, const float* type0,
                  const float* gamma, const float* beta, float eps, int n, int S, int w, int vocab, float* x,
                  __nv_bfloat16* h, int32_t* kv_len, cudaStream_t s);

// RoBERTa-style embeddings (MPNet, XLM-R): x = LN(word[ids] (+ token_type[0]) + position[p]) with HF's position rule
// p = pad + (non-pad ids among ids[b, 0..s]) for a non-pad id and p = pad for a pad id; type0 NULL (MPNet) adds no
// token-type row.  fp32 + bf16 copies.  kv_len[b] = sum(mask[b, :]) as above.
int roberta_embed_ln(const int32_t* ids, const int32_t* mask, const float* word, const float* pos, const float* type0,
                     const float* gamma, const float* beta, float eps, int n, int S, int w, int vocab, int pad, float* x,
                     __nv_bfloat16* h, int32_t* kv_len, cudaStream_t s);

// CLIP head: for image b take token row (b * S + row_in_seq[b]) (row_in_seq NULL -> 0), LayerNorm it, multiply by
// proj [w, E] (fp32), optionally divide by the L2 norm (no epsilon: abstract_clip_model.py:83-85).
// pooled_ws: fp32 workspace [n, w].  Three kernels with normalize, two without.
int clip_head(const float* x, int S, const int32_t* row_in_seq, const float* gamma, const float* beta, float eps,
              const float* proj, int n, int w, int E, int normalize, float* out, float* pooled_ws, cudaStream_t s);

// BERT head: masked mean over the first kv_len[b] tokens (pool == 0) or the [CLS] row (pool == 1), then
// x / max(|x|, 1e-12) if normalize (F.normalize, hugging_face_model.py:194-195).  kv_len is clamped to [0, S]; 0 gives
// a NaN row under mean pooling, as the reference's sum / mask.sum() does.
int bert_head(const float* x, const int32_t* kv_len, int n, int S, int w, int pool, int normalize, float* out,
              cudaStream_t s);

void f32_to_bf16(const float* src, __nv_bfloat16* dst, long long n, cudaStream_t s);
// conv1.weight [w, 3*p*p] -> bf16 [w, kpad] zero padded
void pad_rows_to_bf16(const float* src, int rows, int k, int kpad, __nv_bfloat16* dst, cudaStream_t s);

// conv1.weight [w, 3, p, p] (fp32) -> bf16 [w, p * kbpd * 64] in the gather GEMM's K order (gemm.cuh: PatchGather):
// k' = dy * (64 * kbpd) + dx * 3 + c; the slots past 3 * p of every pixel row are zero.
void patch_weight_rows(const float* src, int rows, int p, int kbpd, __nv_bfloat16* dst, cudaStream_t s);

// PIL-compatible antialiased bicubic resize (shortest side -> S) + centre crop, uint8 HWC in/out: a horizontal and a
// vertical pass, two kernels.
int resize_crop_u8(const uint8_t* src, int n, int h, int w, int S, uint8_t* dst, cudaStream_t s);
// The same resampling squashed to S x S (x and y scaled independently, no crop): PIL resize((S, S), BICUBIC).
int resize_squash_u8(const uint8_t* src, int n, int h, int w, int S, uint8_t* dst, cudaStream_t s);

// Single-query attention pooling, one query per head: out[b, h*64 .. h*64+63] = softmax_s(q_h . k_{b,s} / 8) v_{b,s}
// (bf16).  q fp32, image b's query at q + b * q_stride: q_stride 0 shares one query (SigLIP's latent), W gives one per
// image (the ResNet attention pool's mean token); kv bf16 [n*S, 2W] (K columns, then V columns, head-major); head_dim 64.
int map_attention(const float* q, long long q_stride, const __nv_bfloat16* kv, int n, int S, int W, int heads,
                  __nv_bfloat16* out, cudaStream_t s);

// ResNet stem conv1 (3 x 3, stride 2, padding 1, 3 input channels) as an im2col A matrix: bf16 [n * (S/2)^2, 64], row =
// output pixel, k = (3 ky + kx) * 3 + c, zero for k >= 27.  Input: uint8 HWC [n, S, S, 3] normalised as the patch
// gather does (u8 != NULL), or already-normalised fp32 CHW [n, 3, S, S].  Taps outside the image are 0.
int stem_im2col(const uint8_t* u8, const float* chw, int n, int S, const float* mean, const float* std,
                __nv_bfloat16* out, cudaStream_t s);
// AvgPool2d(2) over NHWC bf16 [n, H, W, C] -> [n, H/2, W/2, C] (H, W even, C % 8 == 0).
int avgpool2_nhwc(const __nv_bfloat16* in, int n, int H, int W, int C, __nv_bfloat16* out, cudaStream_t s);
// ResNet attention-pool tokens: x NHWC bf16 [n, HW, C] -> out bf16 [n * (HW + 1), C], row 0 of image b = mean_s x_s +
// pos[0], row 1 + s = x_s + pos[1 + s]; pos fp32 [HW + 1, C].
int attnpool_tokens(const __nv_bfloat16* x, const float* pos, int n, int HW, int C, __nv_bfloat16* out, cudaStream_t s);

// out[b] = src[b] / |src[b]| if normalize (no epsilon: abstract_clip_model.py:83-85), else src[b]; rows of E floats.
int l2_rows(const float* src, int n, int E, int normalize, float* out, cudaStream_t s);

// ConvNeXt image tower, over fp32 NHWC x [n, H, W, C] with C a multiple of 64, <= 3072; every LayerNorm is over the C
// channels of one pixel.
// Block head: 7 x 7 depthwise conv (zero padding 3) with bias, w49 fp32 [49, C] (tap 7 dy + dx major), then LayerNorm
// -> bf16 out [n * H * W, C], the fc1 GEMM's A operand.
int dwconv7_ln(const float* x, int n, int H, int W, int C, const float* w49, const float* bias, const float* gamma,
               const float* beta, float eps, __nv_bfloat16* out, cudaStream_t s);
// LayerNorm of every pixel, to exactly one of: out_f32 fp32 [n * H * W, C] (may be x: the stem's norm), or out_patch
// bf16 [n * (H/2) * (W/2), 4C], the 2 x 2 stride-2 downsample conv's GEMM rows, column ((y % 2) * 2 + x % 2) * C + c.
int ln_pixels(const float* x, int n, int H, int W, int C, const float* gamma, const float* beta, float eps,
              float* out_f32, __nv_bfloat16* out_patch, cudaStream_t s);
// Mean over each image's HW pixels of x fp32 [n, HW, C], then LayerNorm -> bf16 out [n, C].
int pool_ln(const float* x, int n, int HW, int C, const float* gamma, const float* beta, float eps, __nv_bfloat16* out,
            cudaStream_t s);

}  // namespace kernels
}  // namespace mb
