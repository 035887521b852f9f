// Hopper flash attention for S >= 128 (attention.cuh).  One CTA per (64 queries, head, sequence):
//   warp 4      TMA producer: the Q tile once, then K and V tiles of 128 keys into a two-stage ring (mbarrier
//               full / empty pairs), all straight from the packed qkv matrix with the 128-byte swizzle;
//   warps 0-3   one MMA warpgroup: S = Q K^T with wgmma m64n128k16 (both operands K-major in smem), the online softmax
//               (attention.cuh: OnlineSoftmax) on the accumulator registers, then O += P V with
//               wgmma m64n{HD}k16 taking P from registers (bf16, the m16n8k16 A fragment the S accumulator layout maps
//               to) and V as the transposed (MN-major) B operand.
// The head dim HD (32, 64, 96 or 128) is a template parameter.  A tile's HD columns are stored as one or two column blocks
// (Tiles), each its own TMA box: block 0 holds the first min(HD, 64) columns, block 1 the HD - 64 after them (HD 96:
// 32, HD 128: 64).  A block of 64 columns (128-byte rows) uses the 128-byte swizzle and one of 32 the 64-byte one, in
// the tensor maps and in the wgmma descriptors alike.  QK^T takes each 16-column k-step from the block it falls in;
// P V issues one wgmma per block, each into its own columns of O.
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
    static constexpr int C0 = HD < 64 ? HD : 64;   // columns of block 0
    static constexpr int C1 = HD - C0;             // columns of block 1 (0: none)
    static constexpr int NB = C1 > 0 ? 2 : 1;      // column blocks
    static constexpr uint32_t Q_BYTES = BQ * HD * 2;
    static constexpr uint32_t Q1_OFFSET = BQ * C0 * 2;       // block 1 of the Q tile
    static constexpr uint32_t KV_TILE_BYTES = BKV * HD * 2;
    static constexpr uint32_t KV1_OFFSET = BKV * C0 * 2;     // block 1 of a K / V tile
    static constexpr uint32_t STAGE_BYTES = 2 * KV_TILE_BYTES;   // K then V
    static constexpr size_t SMEM_BYTES = Q_BYTES + KV_STAGES * STAGE_BYTES + 1024 /*align*/ + 64 /*barriers*/;
    // every block starts on a multiple of the 128-byte swizzle's 1024-byte atom
    static_assert(Q1_OFFSET % 1024 == 0 && Q_BYTES % 1024 == 0 && KV1_OFFSET % 1024 == 0 && KV_TILE_BYTES % 1024 == 0);
};

// The TMA descriptors of the Q tiles and of the K / V tiles, one pair per column block
template <int HD>
struct TensorMaps {
    CUtensorMap q[Tiles<HD>::NB], kv[Tiles<HD>::NB];
};

// K-major descriptor of a Q / K column block, and MN-major descriptor of a V column block, of C columns: the swizzle
// that goes with C
template <int C>
__device__ __forceinline__ uint64_t desc_k(uint32_t smem_addr) {
    if constexpr (C == 64) return ptx::make_desc_k_sw128(smem_addr);
    else return ptx::make_desc_k_sw64(smem_addr);
}
template <int C>
__device__ __forceinline__ uint64_t desc_mn(uint32_t smem_addr) {
    if constexpr (C == 64) return ptx::make_desc_mn_sw128(smem_addr, 0);
    else return ptx::make_desc_mn_sw64(smem_addr, 0);
}

// O[64 x C] += P[64 x 16] V[16 x C]: C columns of O, one column block of V
template <int C>
__device__ __forceinline__ void wgmma_pv(float (&o)[C / 2], const uint32_t (&a)[4], uint64_t desc_v) {
    if constexpr (C == 64) ptx::wgmma_m64n64k16_bf16_rs_tb(o, a, desc_v, 1u);
    else ptx::wgmma_m64n32k16_bf16_rs_tb(o, a, desc_v, 1u);
}

// bytes of the relative-bias band behind the barriers: one float per key of the CTA's key tiles, plus BQ - 1
inline size_t bias_band_bytes(int S) { return ((size_t)(S + BKV - 1) / BKV * BKV + BQ) * sizeof(float); }

// BIAS: add the relative-position bias (attention.cuh: RelBias) to the logits, read from a band of the head's bias row
// staged in shared memory behind the barriers.
template <int HD, int MASK, bool BIAS>
__global__ void __launch_bounds__(THREADS)
attention_wgmma_kernel(const __grid_constant__ TensorMaps<HD> tmaps, __nv_bfloat16* __restrict__ out, int S, int W,
                       const int32_t* __restrict__ kv_len, float scale_log2e, const float* __restrict__ rel_bias,
                       int bias_smax) {
    using T = Tiles<HD>;
    constexpr int C0 = T::C0, C1 = T::C1;
    constexpr uint32_t Q_BYTES = T::Q_BYTES;
    constexpr uint32_t KV_TILE_BYTES = T::KV_TILE_BYTES;
    constexpr uint32_t STAGE_BYTES = T::STAGE_BYTES;
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
            ptx::tma_load_2d(sq, &tmaps.q[0], qfull, h * HD, row0 + q0, ptx::kEvictFirst);
            if constexpr (C1 > 0)
                ptx::tma_load_2d(sq + T::Q1_OFFSET, &tmaps.q[1], qfull, h * HD + C0, row0 + q0, ptx::kEvictFirst);
            for (int j = 0; j < nkb; ++j) {
                const int st = j % KV_STAGES;
                ptx::mbar_wait(&empty[st], ((uint32_t)(j / KV_STAGES) & 1u) ^ 1u);
                ptx::mbar_arrive_expect_tx(&full[st], STAGE_BYTES);
                uint8_t* dst = skv + (size_t)st * STAGE_BYTES;
                ptx::tma_load_2d(dst, &tmaps.kv[0], &full[st], W + h * HD, row0 + j * BKV, ptx::kEvictLast);
                ptx::tma_load_2d(dst + KV_TILE_BYTES, &tmaps.kv[0], &full[st], 2 * W + h * HD, row0 + j * BKV, ptx::kEvictLast);
                if constexpr (C1 > 0) {
                    ptx::tma_load_2d(dst + T::KV1_OFFSET, &tmaps.kv[1], &full[st], W + h * HD + C0, row0 + j * BKV,
                                     ptx::kEvictLast);
                    ptx::tma_load_2d(dst + KV_TILE_BYTES + T::KV1_OFFSET, &tmaps.kv[1], &full[st], 2 * W + h * HD + C0,
                                     row0 + j * BKV, ptx::kEvictLast);
                }
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
        for (int k = 0; k < C0 / 16; ++k)
            ptx::wgmma_m64n128k16_bf16(s, desc_k<C0>(q_base + k * 32), desc_k<C0>(k_base + k * 32), k != 0 ? 1u : 0u);
        if constexpr (C1 > 0) {
#pragma unroll
            for (int k = 0; k < C1 / 16; ++k)
                ptx::wgmma_m64n128k16_bf16(s, desc_k<C1>(q_base + T::Q1_OFFSET + k * 32),
                                           desc_k<C1>(k_base + T::KV1_OFFSET + k * 32), 1u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        uint32_t pa[BKV / 16][4];
        sm.update(s, o, pa, j * BKV);
        // ---- O += P V (64 x HD, K = 128 keys; 16 keys = 16 V rows of C * 2 bytes of each column block per k-step)
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BKV / 16; ++k) {
            wgmma_pv<C0>(*reinterpret_cast<float(*)[C0 / 2]>(o), pa[k], desc_mn<C0>(v_base + k * 32 * C0));
            if constexpr (C1 > 0)
                wgmma_pv<C1>(*reinterpret_cast<float(*)[C1 / 2]>(o + C0 / 2), pa[k],
                             desc_mn<C1>(v_base + T::KV1_OFFSET + k * 32 * C1));
        }
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

// Q tiles of BQ rows and K / V tiles of BKV rows out of the packed qkv matrix, per column block
template <int HD>
TensorMaps<HD> make_tmaps(const __nv_bfloat16* qkv, int B, int S, int W) {
    const uint64_t rows = (uint64_t)B * S;
    TensorMaps<HD> t;
    for (int i = 0; i < Tiles<HD>::NB; ++i) {
        const uint32_t cols = i == 0 ? Tiles<HD>::C0 : Tiles<HD>::C1;
        const CUtensorMapSwizzle swz = cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
        t.q[i] = make_tmap_2d(qkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)3 * W, rows, (uint64_t)3 * W * 2, cols,
                              BQ, swz);
        t.kv[i] = make_tmap_2d(qkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)3 * W, rows, (uint64_t)3 * W * 2,
                               cols, BKV, swz);
    }
    return t;
}

}  // namespace

void launch_wgmma_kernel(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int S, int W, int H, int hd, int mask,
                         const int32_t* kv_len, const RelBias& bias, float scale_log2e, cudaStream_t stream) {
    dispatch<true>(hd, mask, bias.table != nullptr, [&](auto d, auto m, auto with_bias) {
        constexpr int HD = decltype(d)::value, MASK = decltype(m)::value;
        constexpr bool BIAS = decltype(with_bias)::value;
        constexpr size_t BASE = Tiles<HD>::SMEM_BYTES;
        static std::once_flag once;   // one per instantiation
        std::call_once(once, [] {
            MB_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel<HD, MASK, BIAS>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)(BASE + (BIAS ? bias_band_bytes(MAX_BIAS_S) : 0))));
        });
        attention_wgmma_kernel<HD, MASK, BIAS>
            <<<dim3((S + BQ - 1) / BQ, H, B), THREADS, BASE + (BIAS ? bias_band_bytes(S) : 0), stream>>>(
                make_tmaps<HD>(qkv, B, S, W), out, S, W, kv_len, scale_log2e, bias.table, bias.smax);
    });
}

}  // namespace attention
}  // namespace mb
