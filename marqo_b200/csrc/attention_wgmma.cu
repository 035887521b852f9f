// Hopper flash attention for S >= 128 (attention.cuh).  One CTA per (64 queries, head, sequence):
//   warp 4      TMA producer: the Q tile once, then K and V tiles of 128 keys into a two-stage ring (mbarrier
//               full / empty pairs), all straight from the packed qkv matrix with the 128-byte swizzle;
//   warps 0-3   one MMA warpgroup: S = Q K^T with wgmma m64n128k16 (both operands K-major in smem), online softmax in
//               fp32 on the accumulator registers (log2 domain, quad shuffles for the row maxima), then O += P V with
//               wgmma m64n{HD}k16 taking P from registers (bf16, the m16n8k16 A fragment the S accumulator layout maps
//               to) and V as the transposed (MN-major) B operand.
// The head dim HD (32 or 64) is a template parameter.  A Q / K / V row is HD * 2 bytes, so HD = 64 tiles use the 128-byte
// swizzle and HD = 32 tiles the 64-byte one, in the tensor maps and in the wgmma descriptors alike.
// Keys past the sequence's length (S, kv_len[b]) and, for MASK_CAUSAL, past the query are masked to -inf; the tiles TMA
// reads beyond a sequence belong to the next one (or are zero-filled past the matrix) and only ever meet masked scores.
#include <mutex>

#include "attention.cuh"
#include "ptx.cuh"

namespace mb {
namespace attention {

namespace {

constexpr int BQ = 64;
constexpr int BKV = 128;
constexpr int KV_STAGES = 2;
constexpr int THREADS = 160;

template <int HD>
struct Tiles {
    static constexpr uint32_t Q_BYTES = BQ * HD * 2;
    static constexpr uint32_t KV_TILE_BYTES = BKV * HD * 2;
    static constexpr uint32_t STAGE_BYTES = 2 * KV_TILE_BYTES;   // K then V
    static constexpr size_t SMEM_BYTES = Q_BYTES + KV_STAGES * STAGE_BYTES + 1024 /*align*/ + 64 /*barriers*/;
};

// K-major descriptor of a Q / K tile, and MN-major descriptor of a V tile, for the swizzle that goes with HD
template <int HD>
__device__ __forceinline__ uint64_t desc_k(uint32_t smem_addr) {
    if constexpr (HD == 64) return ptx::make_desc_k_sw128(smem_addr);
    else return ptx::make_desc_k_sw64(smem_addr);
}
template <int HD>
__device__ __forceinline__ uint64_t desc_mn(uint32_t smem_addr) {
    if constexpr (HD == 64) return ptx::make_desc_mn_sw128(smem_addr, 0);
    else return ptx::make_desc_mn_sw64(smem_addr, 0);
}

// O[64 x HD] += P[64 x 16] V[16 x HD]
template <int HD>
__device__ __forceinline__ void wgmma_pv(float (&o)[HD / 2], const uint32_t (&a)[4], uint64_t desc_v) {
    if constexpr (HD == 64) ptx::wgmma_m64n64k16_bf16_rs_tb(o, a, desc_v, 1u);
    else ptx::wgmma_m64n32k16_bf16_rs_tb(o, a, desc_v, 1u);
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}

// bytes of the relative-bias band behind the barriers: one float per key of the CTA's key tiles, plus BQ - 1
inline size_t bias_band_bytes(int S) { return ((size_t)(S + BKV - 1) / BKV * BKV + BQ) * sizeof(float); }

// BIAS: add the relative-position bias (attention.cuh: RelBias) to the logits, read from a band of the head's bias row
// staged in shared memory behind the barriers.
template <int HD, int MASK, bool BIAS>
__global__ void __launch_bounds__(THREADS)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv,
                       __nv_bfloat16* __restrict__ out, int S, int W, const int32_t* __restrict__ kv_len,
                       float scale_log2e, const float* __restrict__ rel_bias, int bias_smax) {
    constexpr uint32_t Q_BYTES = Tiles<HD>::Q_BYTES;
    constexpr uint32_t KV_TILE_BYTES = Tiles<HD>::KV_TILE_BYTES;
    constexpr uint32_t STAGE_BYTES = Tiles<HD>::STAGE_BYTES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sq = smem;
    uint8_t* skv = smem + Q_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(skv + KV_STAGES * STAGE_BYTES);
    uint64_t* empty = full + KV_STAGES;
    uint64_t* qfull = empty + KV_STAGES;

    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * BQ;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int len = S;
    if (MASK == MASK_KEYLEN) len = min(S, max(kv_len[b], 0));
    int kend = len;
    if (MASK == MASK_CAUSAL) kend = min(len, q0 + BQ);
    const int nkb = (kend + BKV - 1) / BKV;
    const int row0 = b * S;

    if (threadIdx.x == 0) {
        for (int i = 0; i < KV_STAGES; ++i) {
            ptx::mbar_init(&full[i], 1);
            ptx::mbar_init(&empty[i], 4);   // one arrive per MMA warp
        }
        ptx::mbar_init(qfull, 1);
        ptx::fence_barrier_init();
    }
    float* sbias = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full) + 64);
    if constexpr (BIAS) {   // band entry t: key - query = t - (q0 + BQ - 1)
        const float* row = rel_bias + (size_t)h * (2 * bias_smax - 1);
        for (int t = threadIdx.x; t < nkb * BKV + BQ; t += THREADS) sbias[t] = rel_bias_band_value(row, bias_smax, q0, t);
    }
    __syncthreads();

    if (warp == 4) {
        // ------------------------------------------------------------ TMA producer
        if (lane == 0 && nkb > 0) {
            ptx::mbar_arrive_expect_tx(qfull, Q_BYTES);
            ptx::tma_load_2d(sq, &tmap_q, qfull, h * HD, row0 + q0, ptx::kEvictFirst);
            for (int j = 0; j < nkb; ++j) {
                const int st = j % KV_STAGES;
                ptx::mbar_wait(&empty[st], ((uint32_t)(j / KV_STAGES) & 1u) ^ 1u);
                ptx::mbar_arrive_expect_tx(&full[st], STAGE_BYTES);
                uint8_t* dst = skv + (size_t)st * STAGE_BYTES;
                ptx::tma_load_2d(dst, &tmap_kv, &full[st], W + h * HD, row0 + j * BKV, ptx::kEvictLast);
                ptx::tma_load_2d(dst + KV_TILE_BYTES, &tmap_kv, &full[st], 2 * W + h * HD, row0 + j * BKV, ptx::kEvictLast);
            }
        }
        return;
    }

    // ---------------------------------------------------------------- MMA warpgroup
    const int g = lane >> 2, t = lane & 3;
    const int qrow[2] = {q0 + warp * 16 + g, q0 + warp * 16 + g + 8};
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    float row_max[2] = {-INFINITY, -INFINITY};
    float row_sum[2] = {0.f, 0.f};
    if (nkb > 0) ptx::mbar_wait(qfull, 0);
    const uint32_t q_base = ptx::smem_u32(sq);
    for (int j = 0; j < nkb; ++j) {
        const int st = j % KV_STAGES;
        ptx::mbar_wait(&full[st], (uint32_t)(j / KV_STAGES) & 1u);
        const uint32_t k_base = ptx::smem_u32(skv + (size_t)st * STAGE_BYTES);
        const uint32_t v_base = k_base + KV_TILE_BYTES;
        // ---- S = Q K^T (64 x 128)
        float s[BKV / 2];
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < HD / 16; ++k)
            ptx::wgmma_m64n128k16_bf16(s, desc_k<HD>(q_base + k * 32), desc_k<HD>(k_base + k * 32), k != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        // ---- mask, scale (log2 domain), online softmax
        float mx[2] = {row_max[0], row_max[1]};
#pragma unroll
        for (int i = 0; i < BKV / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = j * BKV + 8 * i + 2 * t + (e & 1);
                const int rr = e >> 1;
                bool ok = key < len;
                if (MASK == MASK_CAUSAL) ok = ok && key <= qrow[rr];
                float v;
                if constexpr (BIAS)
                    v = ok ? s[4 * i + e] * scale_log2e + sbias[key - qrow[rr] + (q0 + BQ - 1)] : -INFINITY;
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
        for (int i = 0; i < HD / 8; ++i) {
            o[4 * i] *= corr[0];
            o[4 * i + 1] *= corr[0];
            o[4 * i + 2] *= corr[1];
            o[4 * i + 3] *= corr[1];
        }
        uint32_t pa[BKV / 16][4];
#pragma unroll
        for (int i = 0; i < BKV / 8; ++i) {
            const float p0 = exp2f(s[4 * i] - msafe[0]), p1 = exp2f(s[4 * i + 1] - msafe[0]);
            const float p2 = exp2f(s[4 * i + 2] - msafe[1]), p3 = exp2f(s[4 * i + 3] - msafe[1]);
            row_sum[0] += p0 + p1;
            row_sum[1] += p2 + p3;
            // k-step i / 2 of P V: keys 8 (i % 2) .. 8 (i % 2) + 7 of its 16
            pa[i >> 1][(i & 1) * 2] = pack_bf16(p0, p1);
            pa[i >> 1][(i & 1) * 2 + 1] = pack_bf16(p2, p3);
        }
        // ---- O += P V (64 x HD, K = 128 keys; 16 keys = 16 V rows of HD * 2 bytes per k-step)
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BKV / 16; ++k) wgmma_pv<HD>(o, pa[k], desc_mn<HD>(v_base + k * 32 * HD));
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty[st]);
    }
    // ---- finalise: O /= row sum (quad-reduced), bf16 stores of the rows that exist
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        row_sum[rr] += __shfl_xor_sync(0xffffffffu, row_sum[rr], 1);
        row_sum[rr] += __shfl_xor_sync(0xffffffffu, row_sum[rr], 2);
    }
    const float inv[2] = {row_sum[0] > 0.f ? 1.f / row_sum[0] : 0.f, row_sum[1] > 0.f ? 1.f / row_sum[1] : 0.f};
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        if (qrow[rr] >= S) continue;
        __nv_bfloat16* dst = out + ((size_t)row0 + qrow[rr]) * W + h * HD + 2 * t;
#pragma unroll
        for (int i = 0; i < HD / 8; ++i)
            *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16(o[4 * i + 2 * rr] * inv[rr], o[4 * i + 2 * rr + 1] * inv[rr]);
    }
}

template <int HD, int MASK>
void launch_mask(const CUtensorMap& tq, const CUtensorMap& tkv, __nv_bfloat16* out, int B, int S, int W, int H,
                 const int32_t* kv_len, cudaStream_t stream) {
    constexpr size_t SMEM_BYTES = Tiles<HD>::SMEM_BYTES;
    static std::once_flag once;
    std::call_once(once, [] {
        MB_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel<HD, MASK, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)SMEM_BYTES));
    });
    const dim3 grid((S + BQ - 1) / BQ, H, B);
    const float scale_log2e = head_scale_log2e(HD);
    attention_wgmma_kernel<HD, MASK, false>
        <<<grid, THREADS, SMEM_BYTES, stream>>>(tq, tkv, out, S, W, kv_len, scale_log2e, nullptr, 0);
}

// Q tiles of BQ rows and K / V tiles of BKV rows out of the packed qkv matrix
template <int HD>
void make_tmaps(const __nv_bfloat16* qkv, int B, int S, int W, CUtensorMap& tq, CUtensorMap& tkv) {
    const uint64_t rows = (uint64_t)B * S;
    const CUtensorMapSwizzle swz = HD == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    tq = make_tmap_2d(qkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)3 * W, rows, (uint64_t)3 * W * 2, HD, BQ, swz);
    tkv = make_tmap_2d(qkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)3 * W, rows, (uint64_t)3 * W * 2, HD, BKV, swz);
}

template <int HD>
void launch_hd(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, int mask,
               const int32_t* kv_len, cudaStream_t stream) {
    CUtensorMap tq, tkv;
    make_tmaps<HD>(qkv, B, S, W, tq, tkv);
    switch (mask) {
        case MASK_NONE: launch_mask<HD, MASK_NONE>(tq, tkv, out, B, S, W, H, kv_len, stream); break;
        case MASK_CAUSAL: launch_mask<HD, MASK_CAUSAL>(tq, tkv, out, B, S, W, H, kv_len, stream); break;
        case MASK_KEYLEN:
            if (!kv_len) fail(B200_ERR_INTERNAL, "attention: kv_len required for key-length masking");
            launch_mask<HD, MASK_KEYLEN>(tq, tkv, out, B, S, W, H, kv_len, stream);
            break;
        default: fail(B200_ERR_INTERNAL, "attention: unknown mask mode %d", mask);
    }
}

}  // namespace

int launch_wgmma(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, int mask,
                 const int32_t* kv_len, cudaStream_t stream) {
    const int hd = head_dim(W, H);
    if (B > 65535) fail(B200_ERR_UNSUPPORTED, "attention: batch %d is too large", B);
    if (hd == 64)
        launch_hd<64>(qkv, out, B, S, W, H, mask, kv_len, stream);
    else
        launch_hd<32>(qkv, out, B, S, W, H, mask, kv_len, stream);
    MB_CUDA(cudaGetLastError());
    return 1;
}

int launch_wgmma_rel_bias(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, const int32_t* kv_len,
                          const RelBias& bias, cudaStream_t stream) {
    constexpr int MAX_S = 1024;   // the shared-memory limit set once below covers the band of S <= MAX_S
    if (B > 65535) fail(B200_ERR_UNSUPPORTED, "attention: batch %d is too large", B);
    if (head_dim(W, H) != 64) fail(B200_ERR_UNSUPPORTED, "attention: the relative bias is built for head_dim 64 only");
    if (S > MAX_S) fail(B200_ERR_UNSUPPORTED, "attention: the relative bias supports sequences of at most %d", MAX_S);
    constexpr size_t BASE = Tiles<64>::SMEM_BYTES;
    static std::once_flag once;
    std::call_once(once, [] {
        MB_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel<64, MASK_KEYLEN, true>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BASE + bias_band_bytes(MAX_S))));
    });
    CUtensorMap tq, tkv;
    make_tmaps<64>(qkv, B, S, W, tq, tkv);
    const dim3 grid((S + BQ - 1) / BQ, H, B);
    attention_wgmma_kernel<64, MASK_KEYLEN, true><<<grid, THREADS, BASE + bias_band_bytes(S), stream>>>(
        tq, tkv, out, S, W, kv_len, head_scale_log2e(64), bias.table, bias.smax);
    MB_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace attention
}  // namespace mb
