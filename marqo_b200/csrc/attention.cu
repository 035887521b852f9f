#include "attention.cuh"

namespace mb {
namespace attention {

constexpr int BQ = 64;        // query rows per CTA (4 warps x 16)
constexpr int BKV = 64;       // keys per block
constexpr int THREADS = 128;
template <int HD>
constexpr int CH_LOG2 = HD == 64 ? 3 : 2;   // log2 of the HD / 8 16-byte chunks per tile row

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

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
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
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

    int len = S;
    if (MASK == MASK_KEYLEN) len = min(S, max(kv_len[b], 0));
    int kend = len;
    if (MASK == MASK_CAUSAL) kend = min(len, q0 + BQ);
    const int nkb = (kend + BKV - 1) / BKV;

    load_tile<HD>(sQ, qbase, q0, S, ld);
    if (nkb > 0) {
        load_tile<HD>(sK[0], kbase, 0, len, ld);
        load_tile<HD>(sV[0], vbase, 0, len, ld);
    }
    cp_async_commit();
    if constexpr (BIAS) {   // band entry t: key - query = t - (q0 + BQ - 1); read after the first block's barrier
        const float* row = rel_bias + (size_t)h * (2 * bias_smax - 1);
        for (int t = threadIdx.x; t < nkb * BKV + BQ; t += THREADS) sBias[t] = rel_bias_band_value(row, bias_smax, q0, t);
    }

    uint32_t qf[HD / 16][4];
    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
    float row_max[2] = {-INFINITY, -INFINITY};
    float row_sum[2] = {0.f, 0.f};
    const int qrow[2] = {q0 + warp * 16 + g, q0 + warp * 16 + g + 8};

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
        float s[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                uint32_t kf[4];
                const int mat = lane >> 3, r = lane & 7;
                ldmatrix_x4(kf, tile_ptr<HD>(sK[buf], np * 16 + (mat >> 1) * 8 + r, ks * 2 + (mat & 1)));
                mma_bf16(s[2 * np], qf[ks], kf[0], kf[1]);
                mma_bf16(s[2 * np + 1], qf[ks], kf[2], kf[3]);
            }
        }
        // ---- mask, scale (log2 domain), online softmax
        float mx[2] = {row_max[0], row_max[1]};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kb * BKV + nt * 8 + 2 * t + (e & 1);
                const int rr = e >> 1;
                bool ok = key < len;
                if (MASK == MASK_CAUSAL) ok = ok && key <= qrow[rr];
                float v;
                if constexpr (BIAS)
                    v = ok ? s[nt][e] * scale_log2e + sBias[key - qrow[rr] + (q0 + BQ - 1)] : -INFINITY;
                else
                    v = ok ? s[nt][e] * scale_log2e : -INFINITY;
                s[nt][e] = v;
                mx[rr] = fmaxf(mx[rr], v);
            }
        }
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
            mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
        }
        float corr[2], msafe[2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            msafe[rr] = mx[rr] == -INFINITY ? 0.f : mx[rr];
            corr[rr] = exp2f(row_max[rr] - msafe[rr]);  // row_max = -inf on the first block -> 0
            row_max[rr] = mx[rr];
            row_sum[rr] *= corr[rr];
        }
#pragma unroll
        for (int nt = 0; nt < HD / 8; ++nt) {
            o[nt][0] *= corr[0];
            o[nt][1] *= corr[0];
            o[nt][2] *= corr[1];
            o[nt][3] *= corr[1];
        }
        float ps[2] = {0.f, 0.f};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float pv = exp2f(s[nt][e] - msafe[e >> 1]);
                s[nt][e] = pv;
                ps[e >> 1] += pv;
            }
        }
        row_sum[0] += ps[0];
        row_sum[1] += ps[1];
        // ---- O += P V
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            uint32_t pa[4];
            pa[0] = pack2(s[2 * ks][0], s[2 * ks][1]);
            pa[1] = pack2(s[2 * ks][2], s[2 * ks][3]);
            pa[2] = pack2(s[2 * ks + 1][0], s[2 * ks + 1][1]);
            pa[3] = pack2(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
            for (int dp = 0; dp < HD / 16; ++dp) {
                uint32_t vf[4];
                const int mat = lane >> 3, r = lane & 7;
                ldmatrix_x4_trans(vf, tile_ptr<HD>(sV[buf], ks * 16 + (mat & 1) * 8 + r, dp * 2 + (mat >> 1)));
                mma_bf16(o[2 * dp], pa, vf[0], vf[1]);
                mma_bf16(o[2 * dp + 1], pa, vf[2], vf[3]);
            }
        }
        __syncthreads();
    }
    if (nkb == 0) {
        cp_async_wait<0>();
        __syncthreads();
    }
    // ---- finalise: O /= rowsum (quad-reduced), stage through sQ (this warp's 16 rows), 16-byte coalesced stores
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        row_sum[rr] += __shfl_xor_sync(0xffffffffu, row_sum[rr], 1);
        row_sum[rr] += __shfl_xor_sync(0xffffffffu, row_sum[rr], 2);
    }
    const float inv[2] = {row_sum[0] > 0.f ? 1.f / row_sum[0] : 0.f, row_sum[1] > 0.f ? 1.f / row_sum[1] : 0.f};
#pragma unroll
    for (int nt = 0; nt < HD / 8; ++nt) {
        const int r0 = warp * 16 + g;
        *reinterpret_cast<uint32_t*>(tile_ptr<HD>(sQ, r0, nt) + 2 * t) = pack2(o[nt][0] * inv[0], o[nt][1] * inv[0]);
        *reinterpret_cast<uint32_t*>(tile_ptr<HD>(sQ, r0 + 8, nt) + 2 * t) = pack2(o[nt][2] * inv[1], o[nt][3] * inv[1]);
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

template <int HD>
void launch_hd(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, int mask, const int32_t* kv_len,
               cudaStream_t stream) {
    const dim3 grid((S + BQ - 1) / BQ, H, B);
    const float scale_log2e = head_scale_log2e(HD);
    switch (mask) {
        case MASK_NONE:
            attention_kernel<HD, MASK_NONE, false>
                <<<grid, THREADS, 0, stream>>>(qkv, out, S, W, kv_len, scale_log2e, nullptr, 0);
            break;
        case MASK_CAUSAL:
            attention_kernel<HD, MASK_CAUSAL, false>
                <<<grid, THREADS, 0, stream>>>(qkv, out, S, W, kv_len, scale_log2e, nullptr, 0);
            break;
        case MASK_KEYLEN:
            if (!kv_len) fail(B200_ERR_INTERNAL, "attention: kv_len required for key-length masking");
            attention_kernel<HD, MASK_KEYLEN, false>
                <<<grid, THREADS, 0, stream>>>(qkv, out, S, W, kv_len, scale_log2e, nullptr, 0);
            break;
        default:
            fail(B200_ERR_INTERNAL, "attention: unknown mask mode %d", mask);
    }
}

int launch(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, int mask, const int32_t* kv_len,
           cudaStream_t stream) {
    if (B <= 0 || S <= 0) return 0;
    if (S >= 128) return launch_wgmma(qkv, out, B, S, W, H, mask, kv_len, stream);
    if (head_dim(W, H) == 64)
        launch_hd<64>(qkv, out, B, S, W, H, mask, kv_len, stream);
    else
        launch_hd<32>(qkv, out, B, S, W, H, mask, kv_len, stream);
    MB_CUDA(cudaGetLastError());
    return 1;
}

int launch_rel_bias(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, const int32_t* kv_len,
                    const RelBias& bias, cudaStream_t stream) {
    if (B <= 0 || S <= 0) return 0;
    if (head_dim(W, H) != 64) fail(B200_ERR_UNSUPPORTED, "attention: the relative bias is built for head_dim 64 only");
    if (!kv_len || !bias.table) fail(B200_ERR_INTERNAL, "attention: the relative bias needs kv_len and a table");
    if (S > bias.smax) fail(B200_ERR_INVALID_ARG, "attention: sequence %d is longer than the bias table (%d)", S, bias.smax);
    if (S >= 128) return launch_wgmma_rel_bias(qkv, out, B, S, W, H, kv_len, bias, stream);
    const dim3 grid((S + BQ - 1) / BQ, H, B);
    attention_kernel<64, MASK_KEYLEN, true>
        <<<grid, THREADS, 0, stream>>>(qkv, out, S, W, kv_len, head_scale_log2e(64), bias.table, bias.smax);
    MB_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace attention
}  // namespace mb
