#include "attention.cuh"
#include "ptx.cuh"

namespace mb {
namespace attention {

constexpr int BKV = 64;       // keys per block
constexpr int THREADS = 128;  // 4 warps x 16 query rows
template <int HD>
constexpr int CH_LOG2 = HD == 64 ? 3 : 2;   // log2 of the HD / 8 16-byte chunks per tile row

using ptx::smem_u32;

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
// d[0..3] (+)= A B: one m16n8 accumulator, chunk d / 4 of a flat accumulator array
__device__ __forceinline__ void mma_bf16(float* d, const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// tile: 64 rows x HD bf16 (HD / 8 16-byte chunks per row), chunks XOR-swizzled so that the 8 rows one ldmatrix reads
// cover all 32 banks: HD = 64 (128 B rows) by (row & 7); HD = 32 (64 B rows, two per 128 B line) by ((row >> 1) & 3).
template <int HD>
__device__ __forceinline__ __nv_bfloat16* tile_ptr(__nv_bfloat16* tile, int row, int chunk) {
    const int swz = HD == 64 ? (row & 7) : ((row >> 1) & 3);
    return tile + row * HD + ((chunk ^ swz) << 3);
}

template <int HD>
__device__ __forceinline__ void load_tile(__nv_bfloat16* tile, const __nv_bfloat16* base, int row0, int nrows, int ld) {
    // base points at (sequence row 0, first column of this head's q/k/v slice)
#pragma unroll
    for (int i = 0; i < (64 << CH_LOG2<HD>) / THREADS; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        const int r = idx >> CH_LOG2<HD>, c = idx & ((1 << CH_LOG2<HD>) - 1);
        const bool ok = row0 + r < nrows;
        const __nv_bfloat16* src = base + (size_t)(ok ? row0 + r : 0) * ld + c * 8;
        cp_async16(tile_ptr<HD>(tile, r, c), src, ok);
    }
}

// BIAS: add the relative-position bias (attention.cuh: RelBias) to the logits.  The kernel serves S < 128, so the
// band of the bias row one CTA meets is at most 2 key blocks + BQ entries.
constexpr int BIAS_BAND = 2 * BKV + BQ;

template <int HD, int MASK, bool BIAS>
__global__ void __launch_bounds__(THREADS)
attention_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int S, int W,
                 const int32_t* __restrict__ kv_len, float scale_log2e, const float* __restrict__ rel_bias,
                 int bias_smax) {
    __shared__ __align__(128) __nv_bfloat16 sQ[BQ * HD];
    __shared__ __align__(128) __nv_bfloat16 sK[2][BKV * HD];
    __shared__ __align__(128) __nv_bfloat16 sV[2][BKV * HD];
    __shared__ float sBias[BIAS ? BIAS_BAND : 1];

    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * BQ;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int ld = 3 * W;
    const __nv_bfloat16* seq = qkv + (size_t)b * S * ld;
    const __nv_bfloat16* qbase = seq + h * HD;
    const __nv_bfloat16* kbase = seq + W + h * HD;
    const __nv_bfloat16* vbase = seq + 2 * W + h * HD;

    const KeyRange kr = key_range<MASK, BKV>(S, kv_len, b, q0);
    const int len = kr.len, nkb = kr.nkb;

    load_tile<HD>(sQ, qbase, q0, S, ld);
    if (nkb > 0) {
        load_tile<HD>(sK[0], kbase, 0, len, ld);
        load_tile<HD>(sV[0], vbase, 0, len, ld);
    }
    cp_async_commit();
    if constexpr (BIAS)   // read after the first block's barrier
        stage_bias_band<BKV, THREADS>(sBias, rel_bias, bias_smax, h, q0, nkb);

    uint32_t qf[HD / 16][4];
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    OnlineSoftmax<MASK, BIAS> sm{{q0 + warp * 16 + g, q0 + warp * 16 + g + 8}, q0, len, scale_log2e, sBias};

    for (int kb = 0; kb < nkb; ++kb) {
        const int buf = kb & 1;
        if (kb + 1 < nkb) {
            load_tile<HD>(sK[buf ^ 1], kbase, (kb + 1) * BKV, len, ld);
            load_tile<HD>(sV[buf ^ 1], vbase, (kb + 1) * BKV, len, ld);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (kb == 0) {
#pragma unroll
            for (int ks = 0; ks < HD / 16; ++ks) {
                const int mat = lane >> 3, r = lane & 7;
                ldmatrix_x4(qf[ks], tile_ptr<HD>(sQ, warp * 16 + (mat & 1) * 8 + r, ks * 2 + (mat >> 1)));
            }
        }
        // ---- S = Q K^T (16 x 64 per warp)
        float s[BKV / 2];
#pragma unroll
        for (int i = 0; i < BKV / 2; ++i) s[i] = 0.f;
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                uint32_t kf[4];
                const int mat = lane >> 3, r = lane & 7;
                ldmatrix_x4(kf, tile_ptr<HD>(sK[buf], np * 16 + (mat >> 1) * 8 + r, ks * 2 + (mat & 1)));
                mma_bf16(s + 8 * np, qf[ks], kf[0], kf[1]);
                mma_bf16(s + 8 * np + 4, qf[ks], kf[2], kf[3]);
            }
        }
        uint32_t pa[BKV / 16][4];
        sm.update(s, o, pa, kb * BKV);
        // ---- O += P V, 16 output columns at a time (fewer registers than k-step by k-step)
#pragma unroll
        for (int dp = 0; dp < HD / 16; ++dp) {
#pragma unroll
            for (int ks = 0; ks < BKV / 16; ++ks) {
                uint32_t vf[4];
                const int mat = lane >> 3, r = lane & 7;
                ldmatrix_x4_trans(vf, tile_ptr<HD>(sV[buf], ks * 16 + (mat & 1) * 8 + r, dp * 2 + (mat >> 1)));
                mma_bf16(o + 8 * dp, pa[ks], vf[0], vf[1]);
                mma_bf16(o + 8 * dp + 4, pa[ks], vf[2], vf[3]);
            }
        }
        __syncthreads();
    }
    if (nkb == 0) {
        cp_async_wait<0>();
        __syncthreads();
    }
    // ---- finalise: O /= row sum, stage through sQ (this warp's 16 rows), 16-byte coalesced stores
    float inv[2];
    sm.finish(inv);
#pragma unroll
    for (int nt = 0; nt < HD / 8; ++nt) {
        const int r0 = warp * 16 + g;
        *reinterpret_cast<uint32_t*>(tile_ptr<HD>(sQ, r0, nt) + 2 * t) =
            pack_bf16x2(o[4 * nt] * inv[0], o[4 * nt + 1] * inv[0]);
        *reinterpret_cast<uint32_t*>(tile_ptr<HD>(sQ, r0 + 8, nt) + 2 * t) =
            pack_bf16x2(o[4 * nt + 2] * inv[1], o[4 * nt + 3] * inv[1]);
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < HD / 16; ++i) {
        const int idx = lane + i * 32;
        const int r = warp * 16 + (idx >> CH_LOG2<HD>), c = idx & ((1 << CH_LOG2<HD>) - 1);
        const int tok = q0 + r;
        if (tok < S) {
            const uint4 val = *reinterpret_cast<const uint4*>(tile_ptr<HD>(sQ, r, c));
            *reinterpret_cast<uint4*>(out + ((size_t)b * S + tok) * W + h * HD + c * 8) = val;
        }
    }
}

int launch(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, int mask, const int32_t* kv_len,
           const RelBias& bias, cudaStream_t stream, int model_hd) {
    if (B <= 0 || S <= 0) return 0;
    const int hd = head_dim(W, H);
    if (hd > 64 && S < 128)
        fail(B200_ERR_UNSUPPORTED, "attention: head_dim %d runs sequences of at least 128 tokens (S = %d)", hd, S);
    if (model_hd < 0 || model_hd > hd)
        fail(B200_ERR_INVALID_ARG, "attention: model head_dim %d does not fit kernel head_dim %d", model_hd, hd);
    const float scale_log2e = head_scale_log2e(model_hd ? model_hd : hd);
    if (bias.table) {
        if (hd != 64 || mask != MASK_KEYLEN)
            fail(B200_ERR_UNSUPPORTED, "attention: the relative bias is built for head_dim 64 with the key-length mask");
        if (S > bias.smax)
            fail(B200_ERR_INVALID_ARG, "attention: sequence %d is longer than the bias table (%d)", S, bias.smax);
        if (S > MAX_BIAS_S)
            fail(B200_ERR_UNSUPPORTED, "attention: the relative bias supports sequences of at most %d", MAX_BIAS_S);
    }
    if (B > 65535) fail(B200_ERR_UNSUPPORTED, "attention: batch %d is too large", B);
    if (mask != MASK_NONE && mask != MASK_CAUSAL && mask != MASK_KEYLEN)
        fail(B200_ERR_INTERNAL, "attention: unknown mask mode %d", mask);
    if (mask == MASK_KEYLEN && !kv_len) fail(B200_ERR_INTERNAL, "attention: kv_len required for key-length masking");
    if (S >= 128) {
        launch_wgmma_kernel(qkv, out, B, S, W, H, hd, mask, kv_len, bias, scale_log2e, stream);
    } else {
        dispatch<false>(hd, mask, bias.table != nullptr, [&](auto d, auto m, auto with_bias) {
            constexpr int HD = decltype(d)::value, MASK = decltype(m)::value;
            constexpr bool BIAS = decltype(with_bias)::value;
            attention_kernel<HD, MASK, BIAS><<<dim3((S + BQ - 1) / BQ, H, B), THREADS, 0, stream>>>(
                qkv, out, S, W, kv_len, scale_log2e, bias.table, bias.smax);
        });
    }
    MB_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace attention
}  // namespace mb
