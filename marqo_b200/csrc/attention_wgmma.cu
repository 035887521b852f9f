// Hopper flash attention for S >= 128 (attention.cuh).  One CTA per (64 queries, head, sequence):
//   warp 4      TMA producer: the Q tile once, then K and V tiles of 128 keys into a two-stage ring (mbarrier
//               full / empty pairs), all straight from the packed qkv matrix with the 128-byte swizzle;
//   warps 0-3   one MMA warpgroup: S = Q K^T with wgmma m64n128k16 (both operands K-major in smem), the online softmax
//               (attention.cuh: OnlineSoftmax) on the accumulator registers, then O += P V with
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
    const KeyRange kr = key_range<MASK, BKV>(S, kv_len, b, q0);
    const int nkb = kr.nkb;
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
    if constexpr (BIAS) stage_bias_band<BKV, THREADS>(sbias, rel_bias, bias_smax, h, q0, nkb);
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
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    OnlineSoftmax<MASK, BIAS> sm{{q0 + warp * 16 + g, q0 + warp * 16 + g + 8}, q0, kr.len, scale_log2e, sbias};
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
        uint32_t pa[BKV / 16][4];
        sm.update(s, o, pa, j * BKV);
        // ---- O += P V (64 x HD, K = 128 keys; 16 keys = 16 V rows of HD * 2 bytes per k-step)
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BKV / 16; ++k) wgmma_pv<HD>(o, pa[k], desc_mn<HD>(v_base + k * 32 * HD));
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty[st]);
    }
    // ---- finalise: O /= row sum, bf16 stores of the rows that exist
    float inv[2];
    sm.finish(inv);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        if (sm.qrow[rr] >= S) continue;
        __nv_bfloat16* dst = out + ((size_t)row0 + sm.qrow[rr]) * W + h * HD + 2 * t;
#pragma unroll
        for (int i = 0; i < HD / 8; ++i)
            *reinterpret_cast<uint32_t*>(dst + 8 * i) =
                pack_bf16x2(o[4 * i + 2 * rr] * inv[rr], o[4 * i + 2 * rr + 1] * inv[rr]);
    }
}

// Q tiles of BQ rows and K / V tiles of BKV rows out of the packed qkv matrix
template <int HD>
void make_tmaps(const __nv_bfloat16* qkv, int B, int S, int W, CUtensorMap& tq, CUtensorMap& tkv) {
    const uint64_t rows = (uint64_t)B * S;
    const CUtensorMapSwizzle swz = HD == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    tq = make_tmap_2d(qkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)3 * W, rows, (uint64_t)3 * W * 2, HD, BQ, swz);
    tkv = make_tmap_2d(qkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)3 * W, rows, (uint64_t)3 * W * 2, HD, BKV, swz);
}

}  // namespace

void launch_wgmma_kernel(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, int hd, int mask,
                         const int32_t* kv_len, const RelBias& bias, cudaStream_t stream) {
    dispatch(hd, mask, bias.table != nullptr, [&](auto d, auto m, auto with_bias) {
        constexpr int HD = decltype(d)::value, MASK = decltype(m)::value;
        constexpr bool BIAS = decltype(with_bias)::value;
        constexpr size_t BASE = Tiles<HD>::SMEM_BYTES;
        static std::once_flag once;   // one per instantiation
        std::call_once(once, [] {
            MB_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel<HD, MASK, BIAS>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)(BASE + (BIAS ? bias_band_bytes(MAX_BIAS_S) : 0))));
        });
        CUtensorMap tq, tkv;
        make_tmaps<HD>(qkv, B, S, W, tq, tkv);
        attention_wgmma_kernel<HD, MASK, BIAS>
            <<<dim3((S + BQ - 1) / BQ, H, B), THREADS, BASE + (BIAS ? bias_band_bytes(S) : 0), stream>>>(
                tq, tkv, out, S, W, kv_len, head_scale_log2e(HD), bias.table, bias.smax);
    });
}

}  // namespace attention
}  // namespace mb
