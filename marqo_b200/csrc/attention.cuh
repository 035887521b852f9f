// Multi-head attention over packed QKV (head_dim 32 or 64; 96 or 128 for S >= 128), flash-style online softmax in fp32,
// one CTA per (64 queries, head, sequence).  launch() validates the arguments once and picks the kernel:
//   S >= 128: wgmma kernel (attention_wgmma.cu) — TMA-fed 128-key K / V tiles, one MMA warpgroup, P from registers.
//   S <  128: warp-level kernel (attention.cu, mma.sync m16n8k16, 64-key blocks) — a ViT-B-32 (50 tokens) or CLIP text
//             (77 tokens) sequence would leave 40-60 % of a 128-key wgmma tile masked.
// Head dims 96 and 128 serve the ViT-H / g / bigG vision towers (257 or 730 tokens), whose heads of 80, 88 and 104
// columns the model pads with zero columns (model.cu: pad_heads); the logits keep the model head dim's scale.
// Both kernels hold the scores in the same register layout and run the online softmax below on it (OnlineSoftmax); each
// keeps only its data movement, its MMAs and its output stores.
#pragma once
#include <cmath>
#include <type_traits>

#include "common.cuh"

namespace mb {
namespace attention {

enum Mask { MASK_NONE = 0, MASK_CAUSAL = 1, MASK_KEYLEN = 2 };

constexpr int BQ = 64;   // query rows per CTA, both kernels

// Additive relative-position bias of the attention logits (MPNet): table fp32 [H][2 * smax - 1], already multiplied by
// log2(e); query i and key j of head h add table[h][j - i + smax - 1] to their log2-domain logit.  Each CTA stages the
// diagonal band its 64 queries reach in shared memory.  Built for head_dim 64 with MASK_KEYLEN only; S <= smax and
// S <= MAX_BIAS_S.  An empty table means no bias.
struct RelBias {
    const float* table = nullptr;
    int smax = 0;
};
constexpr int MAX_BIAS_S = 1024;   // the wgmma kernel's shared-memory limit covers the band of up to this many keys

// qkv: bf16 [B*S, 3*W] rows = tokens, columns = [q | k | v], head h occupies columns h*D..h*D+D-1 of each part, where
// D = W / H is the kernel head dim, 32 or 64 (either kernel) or 96 or 128 (S >= 128); the kernels take it as the
// compile-time parameter HD.  model_hd: the head dim whose 1 / sqrt scales the logits, when the heads carry zero pad
// columns up to D; 0 means D.
// out: bf16 [B*S, W].  kv_len: int32 [B] valid key count per sequence (MASK_KEYLEN only).
// Errors: a head dim other than 32 / 64 / 96 / 128, head dim 96 / 128 with S < 128, B > 65535 (gridDim.z), a bias
// without head_dim 64 and MASK_KEYLEN or with S > MAX_BIAS_S: B200_ERR_UNSUPPORTED; a bias with S > smax or a model_hd
// outside 1..D: B200_ERR_INVALID_ARG; an unknown mask or MASK_KEYLEN without kv_len: B200_ERR_INTERNAL.  Returns the
// number of kernels launched.
int launch(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, int mask, const int32_t* kv_len,
           const RelBias& bias, cudaStream_t stream, int model_hd = 0);

// The wgmma kernel's launch (attention_wgmma.cu), for arguments launch() has validated; launch() runs it for S >= 128.
void launch_wgmma_kernel(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, int hd, int mask,
                         const int32_t* kv_len, const RelBias& bias, float scale_log2e, cudaStream_t stream);

// W / H when it is a head dim the kernels are built for (32, 64, 96 or 128); anything else fails with
// B200_ERR_UNSUPPORTED.
inline int head_dim(int W, int H) {
    for (int hd : {64, 32, 96, 128})
        if (H > 0 && W == H * hd) return hd;
    fail(B200_ERR_UNSUPPORTED, "attention: head_dim must be 32, 64, 96 or 128 (width %d, heads %d)", W, H);
}

// softmax scale 1/sqrt(hd), times log2(e): the kernels exponentiate with exp2.  hd 32 and 64 keep their fp32 constants.
inline float head_scale_log2e(int hd) {
    const float scale = hd == 64 ? 0.125f : hd == 32 ? 0.17677669529663687f : (float)(1.0 / std::sqrt((double)hd));
    return scale * 1.4426950408889634f;
}

// Calls f(std::integral_constant<int, HD>, std::integral_constant<int, MASK>, std::bool_constant<BIAS>) for the
// instantiation of (hd, mask, bias) that launch() has accepted: the one list of the instantiations the kernels serve,
// {32, 64} x {none, causal, key length} without the bias, and <64, MASK_KEYLEN, true>; WIDE (the wgmma kernel only)
// adds {96, 128} x {none, causal, key length} without the bias.
template <bool WIDE, class F>
void dispatch(int hd, int mask, bool bias, F&& f) {
    if (bias) return f(std::integral_constant<int, 64>{}, std::integral_constant<int, MASK_KEYLEN>{}, std::true_type{});
    const auto with_mask = [&](auto d) {
        if (mask == MASK_NONE)
            f(d, std::integral_constant<int, MASK_NONE>{}, std::false_type{});
        else if (mask == MASK_CAUSAL)
            f(d, std::integral_constant<int, MASK_CAUSAL>{}, std::false_type{});
        else
            f(d, std::integral_constant<int, MASK_KEYLEN>{}, std::false_type{});
    };
    if constexpr (WIDE) {
        if (hd == 96) return with_mask(std::integral_constant<int, 96>{});
        if (hd == 128) return with_mask(std::integral_constant<int, 128>{});
    }
    if (hd == 64)
        with_mask(std::integral_constant<int, 64>{});
    else
        with_mask(std::integral_constant<int, 32>{});
}

// Keys of sequence b that a CTA whose queries start at q0 attends to: keys >= len are masked, and the key loop runs over
// nkb blocks of BKV keys (MASK_CAUSAL: up to the CTA's last query).
struct KeyRange {
    int len, nkb;
};
template <int MASK, int BKV>
__device__ __forceinline__ KeyRange key_range(int S, const int32_t* __restrict__ kv_len, int b, int q0) {
    int len = S;
    if (MASK == MASK_KEYLEN) len = min(S, max(kv_len[b], 0));
    int kend = len;
    if (MASK == MASK_CAUSAL) kend = min(len, q0 + BQ);
    return {len, (kend + BKV - 1) / BKV};
}

// BIAS: stages the band of head h's bias row that queries q0..q0 + BQ - 1 meet with the keys of nkb blocks of BKV:
// band entry t is key - query = t - (q0 + BQ - 1).  Entries outside the table (never met by a key that is kept) are 0.
template <int BKV, int THREADS>
__device__ __forceinline__ void stage_bias_band(float* band, const float* __restrict__ rel_bias, int smax, int h, int q0,
                                                int nkb) {
    const float* row = rel_bias + (size_t)h * (2 * smax - 1);
    for (int t = threadIdx.x; t < nkb * BKV + BQ; t += THREADS) {
        const int idx = t - (q0 + BQ - 1) + smax - 1;
        band[t] = idx >= 0 && idx < 2 * smax - 1 ? __ldg(row + idx) : 0.f;
    }
}

// Online softmax (fp32, log2 domain) of one warp's 16 query rows over a CTA's key blocks, in the accumulator layout
// mma.sync m16n8 and wgmma m64nN share: with g = lane / 4 and t = lane % 4, a thread holds rows g and g + 8 of its warp's
// 16 (query rows qrow[0], qrow[1]), and 8-column chunk i of an accumulator x holds x[4i], x[4i + 1] (row g) and
// x[4i + 2], x[4i + 3] (row g + 8) at columns 8i + 2t and 8i + 2t + 1.  The scores and O are such accumulators.
template <int MASK, bool BIAS>
struct OnlineSoftmax {
    int qrow[2];
    int q0;                   // the CTA's first query
    int len;                  // keys >= len are masked (key_range)
    float scale_log2e;
    const float* band;        // BIAS: the CTA's bias band in shared memory (stage_bias_band)
    float row_sum[2] = {0.f, 0.f};
    float row_max[2] = {-INFINITY, -INFINITY};

    // One block of keys key0..: s holds its raw scores, NS / 4 chunks of 8 keys.  Masks them (-inf), scales them (plus the
    // bias) into the log2 domain, moves the row maxima (quad shuffles) and rescales row_sum and o by exp2(old - new),
    // then writes the probabilities as bf16 m16n8k16 A fragments, pa[k] for keys 16k..16k + 15 of the block, and adds
    // them to row_sum chunk by chunk.  A row whose keys are all masked keeps a maximum of -inf and gets P = 0.
    template <int NS, int NO>
    __device__ __forceinline__ void update(float (&s)[NS], float (&o)[NO], uint32_t (&pa)[NS / 8][4], int key0) {
        const int t = threadIdx.x & 3;
        float mx[2] = {row_max[0], row_max[1]};
#pragma unroll
        for (int i = 0; i < NS / 4; ++i) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = key0 + 8 * i + 2 * t + (e & 1);
                const int rr = e >> 1;
                bool ok = key < len;
                if (MASK == MASK_CAUSAL) ok = ok && key <= qrow[rr];
                float v;
                if constexpr (BIAS)
                    v = ok ? s[4 * i + e] * scale_log2e + band[key - qrow[rr] + (q0 + BQ - 1)] : -INFINITY;
                else
                    v = ok ? s[4 * i + e] * scale_log2e : -INFINITY;
                s[4 * i + e] = v;
                mx[rr] = fmaxf(mx[rr], v);
            }
        }
        float corr[2], msafe[2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
            mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
            msafe[rr] = mx[rr] == -INFINITY ? 0.f : mx[rr];
            corr[rr] = exp2f(row_max[rr] - msafe[rr]);   // row_max = -inf on the first block -> 0
            row_max[rr] = mx[rr];
            row_sum[rr] *= corr[rr];
        }
#pragma unroll
        for (int i = 0; i < NO / 4; ++i) {
            o[4 * i] *= corr[0];
            o[4 * i + 1] *= corr[0];
            o[4 * i + 2] *= corr[1];
            o[4 * i + 3] *= corr[1];
        }
#pragma unroll
        for (int i = 0; i < NS / 4; ++i) {
            const float p0 = exp2f(s[4 * i] - msafe[0]), p1 = exp2f(s[4 * i + 1] - msafe[0]);
            const float p2 = exp2f(s[4 * i + 2] - msafe[1]), p3 = exp2f(s[4 * i + 3] - msafe[1]);
            row_sum[0] += p0 + p1;
            row_sum[1] += p2 + p3;
            // k-step i / 2 of P V: keys 8 (i % 2) .. 8 (i % 2) + 7 of its 16
            pa[i >> 1][(i & 1) * 2] = pack_bf16x2(p0, p1);
            pa[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(p2, p3);
        }
    }

    // After the last block: the reciprocals of the full row sums (reduced over the quad), 0 for a row without keys.
    __device__ __forceinline__ void finish(float (&inv)[2]) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            row_sum[rr] += __shfl_xor_sync(0xffffffffu, row_sum[rr], 1);
            row_sum[rr] += __shfl_xor_sync(0xffffffffu, row_sum[rr], 2);
        }
        inv[0] = row_sum[0] > 0.f ? 1.f / row_sum[0] : 0.f;
        inv[1] = row_sum[1] > 0.f ? 1.f / row_sum[1] : 0.f;
    }
};

}  // namespace attention
}  // namespace mb
