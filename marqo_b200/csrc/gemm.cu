#include "gemm.cuh"

#include <mutex>
#include <type_traits>

#include "ptx.cuh"

namespace mb {
namespace gemm {

// Two warp-specialised wgmma GEMM kernels share one epilogue: a warpgroup's 64-row output block goes through shared
// memory as 128-byte-wide TMA boxes with the 128B swizzle (the fp32 residual TMA-loaded into the same boxes
// beforehand), the MMA threads write act(acc + bias) (+ residual) over it (epilogue_to_smem), and one thread per
// warpgroup stores the boxes by TMA, which clips them at M and N.  The output type and the activation are template
// parameters of both kernels, so each instantiation holds only the epilogue it runs; the host maps an Epilogue to its
// instantiation in one place (dispatch).
//
// gemm_kernel: one CTA computes a BM x BN = 128 x 128 tile:
//   warps 0-7   two MMA warpgroups, 64 rows of the tile each (wgmma m64n128k16, fp32 accumulators in registers), then
//               the epilogue;
//   warps 8..   the producer: one warp issuing TMA loads of A and W k-blocks (128B swizzle) into a STAGES-deep smem ring,
//               or, for the ViT patch embedding (PROD_PATCH) and the 3 x 3 convolutions (PROD_CONV), four warps that
//               build the A stage from the uint8 image or the NHWC activation while one of them still loads W by TMA.
// Two CTAs share an SM (3 x 32 KB stages each), so one CTA's epilogue overlaps the other's main loop.
// Warpgroup wg's 64 x 128 block of the output goes through one ring stage, the one of virtual k-block kblocks + wg:
// the producer takes that stage through the usual empty/full protocol once the main loop has released it (k-block
// kblocks + wg - 3), and fills it with the fp32 residual rows by TMA when there is a residual, so the load overlaps the
// last MMAs.  The bias columns are read once per CTA into shared memory.
//
// gemm_persistent_kernel: GEMMs with K >= 1024, N % 256 == 0 and at least one full wave of tiles (the ViT-L-14
// layers).  128 x 256 tiles on a persistent grid, one CTA per SM walking the tiles t = blockIdx.x + i * gridDim.x,
// m-major (tile_m = t / tiles_n), so the W columns in use stay in L2.  384 threads:
//   warpgroup 0     the producer: one thread issues the TMA loads into a 3-stage ring of 48 KB; the warpgroup gives its
//                   registers to the MMA warpgroups (setmaxnreg 40).
//   warpgroups 1-2  wgmma m64n256k16 on 64 rows each (128 accumulators per thread, setmaxnreg 232), then the
//                   epilogue through the warpgroup's own EPI_BYTES shared-memory buffer.
//   The ring position `it` is one running counter over every k-block of every tile of the CTA, in the producer and in
//   the MMA warpgroups alike (stage it % 3, phase (it / 3) & 1); it never restarts for a new tile, so the producer runs
//   on into the next tile's k-blocks while the MMA warpgroups are in the epilogue.
//   Per 64-wide k-block a 128 x 256 tile moves 48 KB of TMA writes and 80 KB of wgmma reads through shared memory for
//   4.2 MFLOP, against 32 + 48 KB per 2.1 MFLOP for 128 x 128: its main loop alone runs QKV at 793 TFLOP/s where the
//   same kernel with 128 x 128 tiles reaches 576 (DESIGN.md §7.5c).  With one CTA per SM nothing covers its epilogue,
//   so it pays only where a tile has enough k-blocks; launch() picks it for K >= 1024 and whole 256-wide column tiles.
constexpr int BM = 128;
constexpr int BN = 128;
constexpr int BK = 64;
constexpr int WG_K = 16;
constexpr int STAGES = 3;
constexpr int MMA_THREADS = 256;
constexpr uint32_t A_STAGE_BYTES = BM * BK * 2;
constexpr uint32_t B_STAGE_BYTES = BN * BK * 2;
constexpr uint32_t STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr uint32_t BARRIER_BYTES = 256;
constexpr size_t SMEM_BYTES = (size_t)STAGES * STAGE_BYTES + 1024 /*align*/ + BARRIER_BYTES + 2 * BN * 4 /*bias*/;
// Epilogue: a warpgroup's 64 output rows as 128-byte-wide TMA boxes with the 128B swizzle, 8 KB each, one
// after the other in its stage: fp32 -> 4 boxes of 32 columns (the residual arrives in the same layout), bf16 -> 2
// boxes of 64 columns.
constexpr int EPI_ROWS = BM / 2;
constexpr uint32_t EPI_BOX_BYTES = EPI_ROWS * 128;
static_assert(4 * EPI_BOX_BYTES == STAGE_BYTES, "a warpgroup's fp32 64 x 128 block is one ring stage");

// gemm_persistent_kernel: ring, two epilogue buffers (a warpgroup's bf16 64 x 256 block, or one 128-column half of its
// fp32 block), bias [2][P_BN], barriers
constexpr int P_BN = 256;
constexpr int P_STAGES = 3;
constexpr uint32_t P_STAGE_BYTES = A_STAGE_BYTES + P_BN * BK * 2;
constexpr uint32_t P_RING_BYTES = P_STAGES * P_STAGE_BYTES;
constexpr uint32_t EPI_BYTES = 4 * EPI_BOX_BYTES;
constexpr int PERSISTENT_THREADS = 128 + MMA_THREADS;
constexpr size_t P_SMEM_BYTES = 1024 /*align*/ + P_RING_BYTES + 2 * EPI_BYTES + 2 * P_BN * 4 + BARRIER_BYTES;
static_assert(P_SMEM_BYTES <= 227 * 1024, "over the opt-in shared memory of an H100 CTA");
static_assert(P_BN * 2 * EPI_ROWS == EPI_BYTES, "a warpgroup's bf16 64 x 256 block is one epilogue buffer");

// How gemm_kernel's producer fills the A stages: TMA from an A matrix, or four gather warps building them from the
// uint8 image (ViT patch embedding) or from an NHWC activation (3 x 3 convolution).
enum Producer { PROD_TMA = 0, PROD_PATCH = 1, PROD_CONV = 2 };

template <bool GATHER>
constexpr int threads() { return MMA_THREADS + (GATHER ? 128 : 32); }

struct Params {
    int M, N, K;
    int tiles_m, tiles_n;
    Epilogue ep;
    // PROD_PATCH: uint8 HWC images [n, S, S, 3]; A row r = token t = r % (g*g + cls) of image r / (g*g + cls): zero
    // for t < cls (the class token), else patch t - cls, row-major in the grid.
    // k index of the A row = dy * (64 * kbpd) + dx * 3 + c (kernels::patch_weight_rows lays W out the same way).
    // PROD_CONV (gemm.cuh: ConvGather) reuses four of these fields rather than growing Params, whose layout every
    // other instantiation's code depends on: img is the NHWC bf16 activation [n, H, W, cin], g = H, patch = W and
    // kbpd = cin.
    const uint8_t* img;
    int g;                  // patches per image side
    int patch;              // patch edge in pixels
    int row_bytes;          // 3 * S
    int seg;                // 3 * patch: bytes (= k values) of one patch pixel row
    int kbpd;               // 64-slot k-blocks per patch pixel row: ceil(seg / 64)
    float nscale[3], nshift[3];   // (u8 * nscale[c] + nshift[c]) == (u8/255 - mean[c]) / std[c]
    int cls;                // class-token rows per image: 1 (CLIP) or 0 (SigLIP)
};

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// erf(a) = sign(a) * (1 - exp(P(|a|))) with the single-branch minimax polynomial of the large-argument branch of the
// usual float erf (coefficients pre-multiplied by log2(e) so the exponential is one ex2.approx).  Max abs error of
// erf 1.9e-5, of GELU 1.9e-6 (5.9e-5 relative) — two orders below the bf16 rounding applied to the result
// (tests/test_kernels_gpu.py::test_gemm_epilogues compares against torch's exact erf GELU).
__device__ __forceinline__ float gelu_erf(float x) {
    const float a = x * 0.70710678118654752440f;
    const float t = fabsf(a);
    const float s = a * a;
    float r = fmaf(-2.49374837e-5f, t, 5.52836593e-4f);
    const float u = fmaf(-5.60337594e-3f, t, 3.49920232e-2f);
    r = fmaf(r, s, u);
    r = fmaf(r, t, -1.54047912e-1f);
    r = fmaf(r, t, -9.15890168e-1f);
    r = fmaf(r, t, -1.85700115e-1f);
    r = fmaf(r, t, -1.44269504f * t);
    const float e = copysignf(1.0f - ex2_approx(r), a);
    const float hx = 0.5f * x;
    return fmaf(hx, e, hx);
}

// The same erf-GELU on TWO elements per instruction (HFMA2 / ex2.approx.f16x2), for outputs that are rounded to bf16 anyway
// (fc1's epilogue: the r02 profile had it at 16 fp32 instructions per element and the GEMM epilogue-bound at 75 % tensor
// pipe).  The error is absolute, not relative: fp16 roundings of 2^-11 (of 1 - e, of ex2's argument and result, of the
// final fma) scale with |x| / 2, so the bf16 result y obeys |y - GELU(x)| <= 2^-8 |GELU(x)| + 2^-9 |x| + 2^-24 (bf16
// rounding, fp16 evaluation, fp16 subnormal spacing; tests/test_gemm_shapes_gpu.py::test_activation_edges).  In the
// negative tail that is far from relative: x = -3 gives -0.00439 for -0.00405.  The reference's own CUDA path
// evaluates GELU in fp16 under torch.autocast too (open_clip_model.py:256-258).  Past |x| = 360 a * a overflows to
// inf and the result is x or 0, as it should be; |x| >= 65520 is an fp16 infinity, which act() keeps away from here.
__device__ __forceinline__ __half2 gelu_erf_h2(__half2 x) {
    const __half2 a = __hmul2(x, __float2half2_rn(0.70710678118654752440f));
    const __half2 t = __habs2(a);
    const __half2 s = __hmul2(a, a);
    __half2 r = __hfma2(__float2half2_rn(-2.49374837e-5f), t, __float2half2_rn(5.52836593e-4f));
    const __half2 u = __hfma2(__float2half2_rn(-5.60337594e-3f), t, __float2half2_rn(3.49920232e-2f));
    r = __hfma2(r, s, u);
    r = __hfma2(r, t, __float2half2_rn(-1.54047912e-1f));
    r = __hfma2(r, t, __float2half2_rn(-9.15890168e-1f));
    r = __hfma2(r, t, __float2half2_rn(-1.85700115e-1f));
    r = __hfma2(r, t, __hmul2(t, __float2half2_rn(-1.44269504f)));
    const __half2 e = h2exp2(r);
    const __half2 om = __hsub2(__float2half2_rn(1.0f), e);
    // copysign(1 - e, a) on both halves
    const uint32_t eb = (*reinterpret_cast<const uint32_t*>(&om) & 0x7fff7fffu) | (*reinterpret_cast<const uint32_t*>(&a) & 0x80008000u);
    const __half2 erfv = *reinterpret_cast<const __half2*>(&eb);
    const __half2 hx = __hmul2(x, __float2half2_rn(0.5f));
    return __hfma2(hx, erfv, hx);
}

__device__ __forceinline__ float quick_gelu(float x) {   // x * sigmoid(1.702 x)
    return x / (1.0f + ex2_approx(-1.702f * 1.44269504f * x));
}

// Offset of bf16 element (row, k) inside a 128-row x 64-column K-major stage with the 128-byte swizzle TMA applies:
// 16-byte unit u of row r lands at unit u ^ (r & 7).
__device__ __forceinline__ uint32_t sw128_offset(int row, int unit) {
    return (uint32_t)row * 128u + (uint32_t)((unit ^ (row & 7)) << 4);
}

// Offset of element (row, col) of a warpgroup's staged 64 x 128 block (EPI_BOX_BYTES boxes of 128 / ELEM columns).  A
// warp's store of one fragment (8 rows x 4 column pairs) touches 8 different 16-byte units per row phase: no bank
// conflicts.
template <int ELEM>
__device__ __forceinline__ uint32_t epi_offset(int row, int col) {
    constexpr int BOX_COLS = 128 / ELEM;
    const int byte = (col % BOX_COLS) * ELEM;
    return (uint32_t)(col / BOX_COLS) * EPI_BOX_BYTES + sw128_offset(row, byte >> 4) + (uint32_t)(byte & 15);
}

// Named barrier over the 128 threads of MMA warpgroup wg (ids 1 and 2; 0 is __syncthreads).
__device__ __forceinline__ void warpgroup_sync(int wg) {
    if (wg == 0)
        ptx::bar_sync<1, 128>();
    else
        ptx::bar_sync<2, 128>();
}

// The activation of an adjacent column pair.  A bf16 output (QKV, fc1) evaluates erf-GELU on packed fp16 pairs (see
// gelu_erf_h2), an fp32 output in fp32.
template <bool OUT_FP32, int ACT>
__device__ __forceinline__ float2 act(float x0, float x1) {
    if constexpr (ACT == ACT_GELU && !OUT_FP32) {
        // |x| >= 65520 rounds to an fp16 infinity, which gelu_erf_h2 turns into +inf or NaN; beyond the fp16 range
        // GELU(x) is x or -0 to far better than bf16 precision, so those elements take it in fp32
        float2 y = __half22float2(gelu_erf_h2(__floats2half2_rn(x0, x1)));
        y.x = x0 >= 65504.f ? x0 : x0 <= -65504.f ? -0.f : y.x;
        y.y = x1 >= 65504.f ? x1 : x1 <= -65504.f ? -0.f : y.y;
        return y;
    } else if constexpr (ACT == ACT_GELU)
        return make_float2(gelu_erf(x0), gelu_erf(x1));
    else if constexpr (ACT == ACT_QUICKGELU)
        return make_float2(quick_gelu(x0), quick_gelu(x1));
    else if constexpr (ACT == ACT_RELU)
        return make_float2(fmaxf(x0, 0.f), fmaxf(x1, 0.f));
    else
        return make_float2(x0, x1);
}

// The epilogue of COLS output columns of a warpgroup's 64 rows, held in acc[0, COLS / 2) (fragment i: columns
// 8 i + 2 (lane & 3) + {0, 1} of rows rbase and rbase + 8): act(acc + bias) with the bias row at shared address bias_s,
// plus the fp32 residual already in the buffer when there is one, written at epi_offset into the buffer at shared
// address buf_s.  ACT_RELU (bf16 only) adds its bf16 residual, already in the buffer in the output's layout, before
// the activation.
template <bool OUT_FP32, int ACT, int COLS>
__device__ __forceinline__ void epilogue_to_smem(const float* acc, uint32_t bias_s, uint32_t buf_s, bool residual,
                                                 int rbase, int lane) {
    static_assert(!(OUT_FP32 && ACT == ACT_RELU), "ACT_RELU writes bf16");
#pragma unroll
    for (int i = 0; i < COLS / 8; ++i) {
        const int col = 8 * i + 2 * (lane & 3);
        const float2 bv = ptx::ld_shared_f32x2(bias_s + 4 * col);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = rbase + 8 * h;
            if constexpr (ACT == ACT_RELU) {
                const uint32_t dst = buf_s + epi_offset<2>(r, col);
                float x0 = acc[4 * i + 2 * h] + bv.x, x1 = acc[4 * i + 2 * h + 1] + bv.y;
                if (residual) {
                    const uint32_t rv = ptx::ld_shared_u32(dst);
                    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&rv));
                    x0 += f.x;
                    x1 += f.y;
                }
                const float2 y = act<false, ACT_RELU>(x0, x1);
                ptx::st_shared_u32(dst, pack_bf16x2(y.x, y.y));
                continue;
            }
            float2 y = act<OUT_FP32, ACT>(acc[4 * i + 2 * h] + bv.x, acc[4 * i + 2 * h + 1] + bv.y);
            if constexpr (OUT_FP32) {
                const uint32_t dst = buf_s + epi_offset<4>(r, col);
                if (residual) {   // in the buffer already, where the result goes
                    const float2 rv = ptx::ld_shared_f32x2(dst);
                    y.x += rv.x;
                    y.y += rv.y;
                }
                ptx::st_shared_f32x2(dst, y.x, y.y);
            } else {
                ptx::st_shared_u32(buf_s + epi_offset<2>(r, col), pack_bf16x2(y.x, y.y));
            }
        }
    }
}

// Arrives on bar expecting the fp32 residual boxes of the 64-row, 128-column block at (row0, c0), and TMA-loads them
// into buf.  Only the boxes that overlap [0, M) x [0, N) are loaded, as the others are never stored; a box that
// straddles M is zero-filled past it and still counts all its bytes.
__device__ __forceinline__ void load_residual_boxes(const CUtensorMap* tmap_r, uint64_t* bar, uint8_t* buf, int row0,
                                                    int c0, int M, int N) {
    const int boxes = row0 < M && c0 < N ? min(4, (N - c0) / 32) : 0;
    ptx::mbar_arrive_expect_tx(bar, (uint32_t)boxes * EPI_BOX_BYTES);
    for (int b = 0; b < boxes; ++b)
        ptx::tma_load_2d(buf + b * EPI_BOX_BYTES, tmap_r, bar, c0 + 32 * b, row0, ptx::kEvictNormal);
}

// The same for a bf16 residual (ACT_RELU): boxes of 64 columns, the output's layout.
__device__ __forceinline__ void load_residual_boxes_bf16(const CUtensorMap* tmap_r, uint64_t* bar, uint8_t* buf,
                                                         int row0, int c0, int M, int N) {
    const int boxes = row0 < M && c0 < N ? min(2, (N - c0 + 63) / 64) : 0;
    ptx::mbar_arrive_expect_tx(bar, (uint32_t)boxes * EPI_BOX_BYTES);
    for (int b = 0; b < boxes; ++b)
        ptx::tma_load_2d(buf + b * EPI_BOX_BYTES, tmap_r, bar, c0 + 64 * b, row0, ptx::kEvictNormal);
}

// TMA-stores the 64-row, COLS-column output block at (row0, c0) from its boxes in buf, clipped at M and N, as one bulk
// group.
template <bool OUT_FP32, int COLS>
__device__ __forceinline__ void store_output_boxes(const CUtensorMap* tmap_o, const uint8_t* buf, int row0, int c0,
                                                   int M, int N) {
    constexpr int BOX_COLS = OUT_FP32 ? 32 : 64;
    if (row0 >= M) return;
    for (int b = 0; b * BOX_COLS < COLS && c0 + b * BOX_COLS < N; ++b)
        ptx::tma_store_2d(tmap_o, buf + b * EPI_BOX_BYTES, c0 + b * BOX_COLS, row0);
    ptx::tma_store_commit();
}

// tmap_r / tmap_o: the fp32 residual and the output, boxes of EPI_ROWS rows x 128 bytes.  p is a grid constant so that
// the gather's run-time index into p.nscale / p.nshift reads the parameter space instead of a local copy of p.
template <int PROD, bool OUT_FP32, int ACT>
__global__ void __launch_bounds__(threads<PROD != PROD_TMA>(), PROD != PROD_TMA ? 1 : 2)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_r, const __grid_constant__ CUtensorMap tmap_o,
            const __grid_constant__ Params p) {
    constexpr bool GATHER = PROD != PROD_TMA;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)STAGES * STAGE_BYTES);
    uint64_t* empty = full + STAGES;
    float* bias_s = reinterpret_cast<float*>(smem + (size_t)STAGES * STAGE_BYTES + BARRIER_BYTES);   // [2][BN]

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const int lane = threadIdx.x & 31;
    const int tile_m = blockIdx.x / p.tiles_n, tile_n = blockIdx.x % p.tiles_n;
    const int m0 = tile_m * BM, n0 = tile_n * BN;
    // K need only be a multiple of 8: the last k-block's columns past K are zero-filled by TMA in A and W alike
    const int kblocks = (p.K + BK - 1) / BK;

    if (threadIdx.x == MMA_THREADS) {
        ptx::prefetch_tmap(&tmap_b);
        if (!GATHER) ptx::prefetch_tmap(&tmap_a);
        ptx::prefetch_tmap(&tmap_o);
        if (p.ep.residual) ptx::prefetch_tmap(&tmap_r);
        for (int i = 0; i < STAGES; ++i) {
            ptx::mbar_init(&full[i], GATHER ? 1 + 128 : 1);
            ptx::mbar_init(&empty[i], MMA_THREADS / 32);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (threadIdx.x >= MMA_THREADS) {
        // ------------------------------------------------------------ producer
        const int pt = threadIdx.x - MMA_THREADS;
        if (!GATHER && pt >= 32) return;
        // GATHER: thread pt builds A row pt of every stage: token row m0 + pt, zero (prow == nullptr) for a class token
        const uint8_t* prow = nullptr;
        // PROD_CONV: thread pt builds A row pt, output pixel (b, cy, cx) = m0 + pt; cimg is image b (NULL: row >= M)
        const __nv_bfloat16* cimg = nullptr;
        int cy = 0, cx = 0;
        const int cH = p.g, cW = p.patch, cin = p.kbpd;   // PROD_CONV's meaning of these fields
        if (PROD == PROD_CONV) {
            const int r = m0 + pt;
            if (r < p.M) {
                const int hw = cH * cW;
                const int b = r / hw, rem = r - b * hw;
                cy = rem / cW;
                cx = rem - cy * cW;
                cimg = reinterpret_cast<const __nv_bfloat16*>(p.img) + (size_t)b * hw * cin;
            }
        }
        if (PROD == PROD_PATCH) {
            const int r = m0 + pt;
            const int tokens = p.g * p.g + p.cls;
            const int b = r / tokens, t = r - b * tokens - p.cls;
            if (r < p.M && t >= 0) {
                const int py = t / p.g, px = t - py * p.g;
                prow = p.img + ((size_t)b * p.g * p.patch + (size_t)py * p.patch) * p.row_bytes + (size_t)px * p.patch * 3;
            }
        }
        for (int kb = 0; kb < kblocks; ++kb) {
            const int stage = kb % STAGES;
            const uint32_t phase = (uint32_t)(kb / STAGES) & 1u;
            uint8_t* sa = smem + (size_t)stage * STAGE_BYTES;
            uint8_t* sb = sa + A_STAGE_BYTES;
            ptx::mbar_wait(&empty[stage], phase ^ 1);
            if (pt == 0) {
                ptx::mbar_arrive_expect_tx(&full[stage], GATHER ? B_STAGE_BYTES : STAGE_BYTES);
                if (!GATHER) ptx::tma_load_2d(sa, &tmap_a, &full[stage], kb * BK, m0, ptx::kEvictNormal);
                ptx::tma_load_2d(sb, &tmap_b, &full[stage], kb * BK, n0, ptx::kEvictLast);
            }
            if (PROD == PROD_CONV) {
                // 16-byte unit u holds k = 64 kb + 8 u .. + 7: channels c .. c + 7 of tap t, k = t cin + c.  cin is
                // a multiple of 8, so a unit never straddles two taps: (t, c) walks the k-block in 8-channel steps,
                // onto the next tap whenever c reaches cin (more than once per k-block when cin < 64).  All eight
                // loads are issued before the first store.
                int tap = kb * 64 / cin, c = kb * 64 - tap * cin;
                uint4 v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int iy = cy + tap / 3 - 1, ix = cx + tap % 3 - 1;
                    v[u] = make_uint4(0u, 0u, 0u, 0u);
                    if (cimg != nullptr && tap < 9 && (unsigned)iy < (unsigned)cH && (unsigned)ix < (unsigned)cW)
                        v[u] = __ldg(reinterpret_cast<const uint4*>(cimg + ((size_t)iy * cW + ix) * cin + c));
                    c += 8;
                    if (c == cin) {
                        c = 0;
                        ++tap;
                    }
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) *reinterpret_cast<uint4*>(sa + sw128_offset(pt, u)) = v[u];
                ptx::fence_proxy_async_smem();   // generic-proxy stores -> visible to wgmma's operand reads
                ptx::mbar_arrive(&full[stage]);
            } else if (GATHER) {
                // k-block kb covers k' = dy * 64 kbpd + j0 .. + 63 of the patch's pixel row dy
                const int dy = kb / p.kbpd, j0 = (kb - dy * p.kbpd) * 64;
                const uint8_t* src = prow ? prow + (size_t)dy * p.row_bytes + j0 : nullptr;
                int c = j0 % 3;
#pragma unroll 1
                for (int u = 0; u < 8; ++u) {
                    uint32_t w[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float v[2];
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int j = u * 8 + e * 2 + h;
                            v[h] = (src != nullptr && j0 + j < p.seg) ? fmaf((float)__ldg(src + j), p.nscale[c], p.nshift[c]) : 0.f;
                            c = c == 2 ? 0 : c + 1;
                        }
                        w[e] = pack_bf16x2(v[0], v[1]);
                    }
                    *reinterpret_cast<uint4*>(sa + sw128_offset(pt, u)) = make_uint4(w[0], w[1], w[2], w[3]);
                }
                ptx::fence_proxy_async_smem();   // generic-proxy stores -> visible to wgmma's operand reads
                ptx::mbar_arrive(&full[stage]);
            }
        }
        // virtual k-blocks kblocks, kblocks + 1: the epilogue stages of warpgroups 0 and 1, with their residual rows
        for (int wg = 0; wg < 2; ++wg) {
            const int kb = kblocks + wg;
            const int stage = kb % STAGES;
            uint8_t* s = smem + (size_t)stage * STAGE_BYTES;
            ptx::mbar_wait(&empty[stage], ((uint32_t)(kb / STAGES) & 1u) ^ 1);
            if (pt == 0) {
                if (p.ep.residual != nullptr) {
                    if constexpr (ACT == ACT_RELU)
                        load_residual_boxes_bf16(&tmap_r, &full[stage], s, m0 + EPI_ROWS * wg, n0, p.M, p.N);
                    else
                        load_residual_boxes(&tmap_r, &full[stage], s, m0 + EPI_ROWS * wg, n0, p.M, p.N);
                } else
                    ptx::mbar_arrive(&full[stage]);
            }
            if (GATHER) ptx::mbar_arrive(&full[stage]);   // full[] also counts every gather thread
        }
        return;
    }

    // ---------------------------------------------------------------- MMA warpgroups
    const int wg = warp >> 2;
    const Epilogue& ep = p.ep;
    // thread t of the warpgroup fetches bias column n0 + t now; the load completes under the main loop
    float bias_t = 0.f;
    if (ep.bias != nullptr && n0 + (int)(threadIdx.x & 127) < p.N) bias_t = __ldg(ep.bias + n0 + (threadIdx.x & 127));
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < kblocks; ++kb) {
        const int stage = kb % STAGES;
        ptx::mbar_wait(&full[stage], (uint32_t)(kb / STAGES) & 1u);
        const uint32_t a_base = ptx::smem_u32(smem + (size_t)stage * STAGE_BYTES) + wg * (64 * 128);
        const uint32_t b_base = ptx::smem_u32(smem + (size_t)stage * STAGE_BYTES + A_STAGE_BYTES);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WG_K; ++k)
            ptx::wgmma_m64n128k16_bf16(acc, ptx::make_desc_k_sw128(a_base + k * WG_K * 2),
                                       ptx::make_desc_k_sw128(b_base + k * WG_K * 2), (kb | k) != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();   // the previous k-block's MMAs are done: its stage goes back to the producer
        if (kb > 0 && lane == 0) ptx::mbar_arrive(&empty[(kb - 1) % STAGES]);
    }
    ptx::wgmma_wait<0>();

    // ---------------------------------------------------------------- epilogue through shared memory, TMA store
    const int t = threadIdx.x & 127;
    float* wbias = bias_s + wg * BN;
    wbias[t] = bias_t;
    const int kb = kblocks + wg;
    ptx::mbar_wait(&full[kb % STAGES], (uint32_t)(kb / STAGES) & 1u);   // the stage is ours, the residual in it
    uint8_t* tile = smem + (size_t)(kb % STAGES) * STAGE_BYTES;
    warpgroup_sync(wg);   // wbias complete
    const int rbase = (warp & 3) * 16 + (lane >> 2);   // row inside the warpgroup's 64
    epilogue_to_smem<OUT_FP32, ACT, BN>(acc, ptx::smem_u32(wbias), ptx::smem_u32(tile), ep.residual != nullptr, rbase,
                                        lane);
    ptx::fence_proxy_async_smem();   // generic-proxy stores -> visible to the TMA store
    warpgroup_sync(wg);
    if (t == 0) {
        store_output_boxes<OUT_FP32, BN>(&tmap_o, tile, m0 + EPI_ROWS * wg, n0, p.M, p.N);
        ptx::tma_store_wait_read<0>();   // the stage must outlive the store's reads of it
    }
}

// tmap_r / tmap_o: the fp32 residual (an unused view when there is none) and the output, boxes of EPI_ROWS rows x 128
// bytes.
//
// The epilogue buffer of MMA warpgroup wg is written by three parties, in this order for every use:
//   1. the TMA store of the previous use reads it: issued by thread 0 of the warpgroup (the only thread that stores
//      from it), which is therefore the one that waits for those reads (cp.async.bulk.wait_group.read 0);
//   2. then, with a residual, thread 0 TMA-loads the residual columns of this use into it, completing on epi_full[wg];
//   3. then the 128 threads write act(acc + bias) (+ residual) over it: they wait on epi_full[wg] (residual) or on a
//      warpgroup barrier that thread 0 reaches only after step 1 (no residual); fence.proxy.async and a warpgroup
//      barrier order their writes before thread 0 issues the store of this use.
// Thread 0 waits for the previous tile's last store after it has issued the first k-block of the new tile, so the
// store overlaps the main loop, and the first residual load goes out then too, from L2 (the CTA prefetched the
// tile's second residual half together with its first half).  An fp32 block of P_BN = 256 columns is 64 KB, twice the
// buffer: it goes in two 128-column uses, and the second waits for the first's store inside the epilogue.
// Running in place (residual == out) is safe: the residual rows and columns a tile reads are the ones it writes, and
// no other tile touches them.
// OUT_FP32 and ACT are template parameters so that each instantiation holds only the epilogue it runs: the epilogue is
// unrolled over the 128 accumulators, and with every variant behind runtime branches the kernel was 218 KB of code,
// which each tile's epilogue fetched into a cold instruction cache while the tensor cores idled.
template <bool OUT_FP32, int ACT>
__global__ void __launch_bounds__(PERSISTENT_THREADS, 1)
gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_r, const __grid_constant__ CUtensorMap tmap_o, Params p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* epi_s = smem + P_RING_BYTES;                                // [2][EPI_BYTES]
    float* bias_s = reinterpret_cast<float*>(epi_s + 2 * EPI_BYTES);      // [2][P_BN]
    uint64_t* full = reinterpret_cast<uint64_t*>(bias_s + 2 * P_BN);
    uint64_t* empty = full + P_STAGES;
    uint64_t* epi_full = empty + P_STAGES;                                  // [2]

    const int tiles = p.tiles_m * p.tiles_n;
    const int kblocks = p.K / BK;
    const Epilogue& ep = p.ep;
    const bool has_res = OUT_FP32 && ep.residual != nullptr;

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmap_a);
        ptx::prefetch_tmap(&tmap_b);
        ptx::prefetch_tmap(&tmap_o);
        if (has_res) ptx::prefetch_tmap(&tmap_r);
        for (int i = 0; i < P_STAGES; ++i) {
            ptx::mbar_init(&full[i], 1);
            ptx::mbar_init(&empty[i], MMA_THREADS / 32);
        }
        ptx::mbar_init(&epi_full[0], 1);
        ptx::mbar_init(&epi_full[1], 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (threadIdx.x < 128) {
        // ------------------------------------------------------------ producer
        ptx::setmaxnreg_dec<40>();
        if (threadIdx.x != 0) return;
        uint32_t it = 0;
        for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            const int m0 = (tile / p.tiles_n) * BM, n0 = (tile % p.tiles_n) * P_BN;
            for (int kb = 0; kb < kblocks; ++kb, ++it) {
                const int stage = it % P_STAGES;
                uint8_t* sa = smem + (size_t)stage * P_STAGE_BYTES;
                ptx::mbar_wait(&empty[stage], ((it / P_STAGES) & 1u) ^ 1);
                ptx::mbar_arrive_expect_tx(&full[stage], P_STAGE_BYTES);
                ptx::tma_load_2d(sa, &tmap_a, &full[stage], kb * BK, m0, ptx::kEvictNormal);
                ptx::tma_load_2d(sa + A_STAGE_BYTES, &tmap_b, &full[stage], kb * BK, n0, ptx::kEvictLast);
            }
        }
        return;
    }

    // ---------------------------------------------------------------- MMA warpgroups
    ptx::setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int t = threadIdx.x & 127;
    const int warp = t >> 5, lane = t & 31;
    uint8_t* buf = epi_s + wg * EPI_BYTES;
    float* wbias = bias_s + wg * P_BN;
    const uint32_t buf_s = ptx::smem_u32(buf), wbias_s = ptx::smem_u32(wbias);
    const int rbase = warp * 16 + (lane >> 2);   // row inside the warpgroup's 64
    // columns per use of the buffer: a bf16 block in one use, an fp32 block in two
    constexpr int COLS = OUT_FP32 ? 128 : P_BN;
    uint32_t it = 0, epi_phase = 0;

    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int m0 = (tile / p.tiles_n) * BM, n0 = (tile % p.tiles_n) * P_BN;
        const int row0 = m0 + EPI_ROWS * wg;
        // thread t fetches bias columns n0 + t + 128 j now; the loads complete under the main loop
        float bias_r[P_BN / 128];
#pragma unroll
        for (int j = 0; j < P_BN / 128; ++j) {
            const int c = n0 + t + 128 * j;
            bias_r[j] = ep.bias != nullptr && c < p.N ? __ldg(ep.bias + c) : 0.f;
        }
        float acc[P_BN / 2];
#pragma unroll
        for (int i = 0; i < P_BN / 2; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < kblocks; ++kb, ++it) {
            const int stage = it % P_STAGES;
            ptx::mbar_wait(&full[stage], (it / P_STAGES) & 1u);
            const uint32_t a_base = ptx::smem_u32(smem + (size_t)stage * P_STAGE_BYTES) + wg * (64 * 128);
            const uint32_t b_base = ptx::smem_u32(smem + (size_t)stage * P_STAGE_BYTES + A_STAGE_BYTES);
            ptx::wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / WG_K; ++k) {
                const uint64_t da = ptx::make_desc_k_sw128(a_base + k * WG_K * 2);
                const uint64_t db = ptx::make_desc_k_sw128(b_base + k * WG_K * 2);
                ptx::wgmma_m64n256k16_bf16(acc, da, db, (kb | k) != 0 ? 1u : 0u);
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();   // the previous k-block's MMAs are done: its stage goes back to the producer
            if (kb > 0 && lane == 0) ptx::mbar_arrive(&empty[(it - 1) % P_STAGES]);
            if (kb == 0 && t == 0) {
                ptx::tma_store_wait_read<0>();   // the previous tile's last store has read the buffer
                if (has_res) {
                    load_residual_boxes(&tmap_r, &epi_full[wg], buf, row0, n0, p.M, p.N);
                    if (row0 < p.M)
                        for (int b = 0; b < 4 && n0 + 128 + 32 * b < p.N; ++b)
                            ptx::tma_prefetch_l2_2d(&tmap_r, n0 + 128 + 32 * b, row0);
                }
            }
        }
        ptx::wgmma_wait<0>();
        if (lane == 0) ptx::mbar_arrive(&empty[(it - 1) % P_STAGES]);

        // ------------------------------------------------------------ epilogue through the buffer, TMA store
#pragma unroll
        for (int j = 0; j < P_BN / 128; ++j) wbias[t + 128 * j] = bias_r[j];
        warpgroup_sync(wg);   // wbias complete; without a residual, the buffer is free (thread 0 waited above)
#pragma unroll
        for (int hf = 0; hf < P_BN / COLS; ++hf) {
            if (hf > 0) {   // the buffer holds half hf - 1 until its store has read it
                if (t == 0) {
                    ptx::tma_store_wait_read<0>();
                    if (has_res) load_residual_boxes(&tmap_r, &epi_full[wg], buf, row0, n0 + COLS * hf, p.M, p.N);
                }
                if (!has_res) warpgroup_sync(wg);
            }
            if (has_res) {
                ptx::mbar_wait(&epi_full[wg], epi_phase);
                epi_phase ^= 1;
            }
            epilogue_to_smem<OUT_FP32, ACT, COLS>(acc + COLS / 2 * hf, wbias_s + 4 * COLS * hf, buf_s, has_res, rbase,
                                                  lane);
            ptx::fence_proxy_async_smem();   // generic-proxy stores -> visible to the TMA store
            warpgroup_sync(wg);
            if (t == 0) store_output_boxes<OUT_FP32, COLS>(&tmap_o, buf, row0, n0 + COLS * hf, p.M, p.N);
        }
    }
    if (t == 0) ptx::tma_store_wait_read<0>();   // shared memory must outlive the last store's reads of it
}

// Calls f(std::bool_constant<OUT_FP32>, std::integral_constant<int, ACT>) for the epilogue instantiation of
// (out_fp32, act), an activation other than GELU and QuickGELU being none: the one list of instantiations, from which
// both launches and configure() take theirs.
template <class F>
static void dispatch(bool out_fp32, int act, F&& f) {
    if (act == ACT_RELU) {   // bf16 only (check_epilogue)
        f(std::false_type{}, std::integral_constant<int, ACT_RELU>{});
        return;
    }
    const auto with_act = [&](auto out) {
        if (act == ACT_GELU)
            f(out, std::integral_constant<int, ACT_GELU>{});
        else if (act == ACT_QUICKGELU)
            f(out, std::integral_constant<int, ACT_QUICKGELU>{});
        else
            f(out, std::integral_constant<int, ACT_NONE>{});
    };
    if (out_fp32)
        with_act(std::true_type{});
    else
        with_act(std::false_type{});
}

void configure() {
    static std::once_flag once;
    std::call_once(once, [] {
        const auto attr = cudaFuncAttributeMaxDynamicSharedMemorySize;
        MB_CUDA(cudaFuncSetAttribute(gemm_kernel<PROD_PATCH, true, ACT_NONE>, attr, (int)SMEM_BYTES));
        MB_CUDA(cudaFuncSetAttribute(gemm_kernel<PROD_CONV, false, ACT_RELU>, attr, (int)SMEM_BYTES));
        for (int out_fp32 = 0; out_fp32 < 2; ++out_fp32)
            for (int act = ACT_NONE; act <= ACT_RELU; ++act)
                dispatch(out_fp32, act, [&](auto out, auto a) {
                    constexpr bool OUT_FP32 = decltype(out)::value;
                    constexpr int ACT = decltype(a)::value;
                    MB_CUDA(cudaFuncSetAttribute(gemm_kernel<PROD_TMA, OUT_FP32, ACT>, attr, (int)SMEM_BYTES));
                    MB_CUDA(cudaFuncSetAttribute(gemm_persistent_kernel<OUT_FP32, ACT>, attr, (int)P_SMEM_BYTES));
                });
    });
}

// TMA: 16-byte aligned bases and row pitches
static void check_epilogue(const Epilogue& ep) {
    if (ep.ldo % 8 != 0) fail(B200_ERR_INTERNAL, "gemm: ldo = %d must be a multiple of 8", ep.ldo);
    if ((reinterpret_cast<uintptr_t>(ep.out) & 15) != 0) fail(B200_ERR_INTERNAL, "gemm: output not 16-byte aligned");
    if (ep.act == ACT_RELU && ep.out_fp32) fail(B200_ERR_INTERNAL, "gemm: ReLU writes a bf16 output");
    if (ep.residual != nullptr && (ep.out_fp32 ? ep.ldr % 4 != 0 : ep.act != ACT_RELU || ep.ldr % 8 != 0))
        fail(B200_ERR_INTERNAL, "gemm: the residual needs an fp32 output and ldr %% 4 == 0, or ReLU and ldr %% 8 == 0");
    if (ep.residual != nullptr && (reinterpret_cast<uintptr_t>(ep.residual) & 15) != 0)
        fail(B200_ERR_INTERNAL, "gemm: residual not 16-byte aligned");
}

// The epilogue's maps, boxes of EPI_ROWS rows x 128 bytes with the 128B swizzle: the fp32 residual (tr is left as it
// is without one) and the output.
static void epilogue_tmaps(const Epilogue& ep, int M, int N, CUtensorMap& tr, CUtensorMap& to) {
    if (ep.residual)
        tr = ep.out_fp32 ? make_tmap_2d(ep.residual, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (uint64_t)N, (uint64_t)M,
                                        (uint64_t)ep.ldr * 4, 32, EPI_ROWS, CU_TENSOR_MAP_SWIZZLE_128B)
                         : make_tmap_2d(ep.residual, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)N, (uint64_t)M,
                                        (uint64_t)ep.ldr * 2, 64, EPI_ROWS, CU_TENSOR_MAP_SWIZZLE_128B);
    to = ep.out_fp32 ? make_tmap_2d(ep.out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (uint64_t)N, (uint64_t)M,
                                    (uint64_t)ep.ldo * 4, 32, EPI_ROWS, CU_TENSOR_MAP_SWIZZLE_128B)
                     : make_tmap_2d(ep.out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)N, (uint64_t)M,
                                    (uint64_t)ep.ldo * 2, 64, EPI_ROWS, CU_TENSOR_MAP_SWIZZLE_128B);
}

template <int PROD, bool OUT_FP32, int ACT>
static void launch_tiles(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int M, int N, int K, const Epilogue& ep,
                         cudaStream_t stream, const PatchGather* pg = nullptr, const ConvGather* cg = nullptr) {
    constexpr bool GATHER = PROD != PROD_TMA;
    Params p{};
    if (PROD == PROD_CONV) {   // (Params: the fields PROD_CONV reuses)
        p.img = reinterpret_cast<const uint8_t*>(cg->act);
        p.g = cg->H;
        p.patch = cg->W;
        p.kbpd = cg->cin;
    }
    if (PROD == PROD_PATCH) {
        p.img = pg->img;
        p.patch = pg->patch;
        p.g = pg->S / pg->patch;
        p.row_bytes = 3 * pg->S;
        p.seg = 3 * pg->patch;
        p.kbpd = patch_gather_kbpd(pg->patch);
        p.cls = pg->cls;
        for (int c = 0; c < 3; ++c) {
            p.nscale[c] = (float)(1.0 / (255.0 * (double)pg->std[c]));
            p.nshift[c] = (float)(-(double)pg->mean[c] / (double)pg->std[c]);
        }
    }
    p.M = M;
    p.N = N;
    p.K = K;
    p.tiles_n = (N + BN - 1) / BN;
    p.ep = ep;
    const long long tiles = (long long)((M + BM - 1) / BM) * p.tiles_n;
    if (tiles > 0x7fffffffLL) fail(B200_ERR_UNSUPPORTED, "gemm: %lld tiles is too many", tiles);
    // (GATHER has no A matrix, and without a residual there is no residual map: those maps are further, unused views of
    // W so the kernel signature stays the same)
    CUtensorMap tb = make_tmap_2d(W, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)K, (uint64_t)N, (uint64_t)K * 2, BK, BN,
                                  CU_TENSOR_MAP_SWIZZLE_128B);
    CUtensorMap ta = GATHER ? tb
                            : make_tmap_2d(A, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)K, (uint64_t)M,
                                           (uint64_t)lda * 2, BK, BM, CU_TENSOR_MAP_SWIZZLE_128B);
    CUtensorMap tr = tb, to;
    epilogue_tmaps(ep, M, N, tr, to);
    gemm_kernel<PROD, OUT_FP32, ACT><<<(unsigned)tiles, threads<GATHER>(), SMEM_BYTES, stream>>>(ta, tb, tr, to, p);
    MB_CUDA(cudaGetLastError());
}

template <bool OUT_FP32, int ACT>
static void launch_persistent(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int M, int N, int K,
                              const Epilogue& ep, int sms, cudaStream_t stream) {
    Params p{};
    p.M = M;
    p.N = N;
    p.K = K;
    p.tiles_m = (M + BM - 1) / BM;
    p.tiles_n = (N + P_BN - 1) / P_BN;
    p.ep = ep;
    const long long tiles = (long long)p.tiles_m * p.tiles_n;
    if (tiles > 0x7fffffffLL) fail(B200_ERR_UNSUPPORTED, "gemm: %lld tiles is too many", tiles);
    CUtensorMap ta = make_tmap_2d(A, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2,
                                  BK, BM, CU_TENSOR_MAP_SWIZZLE_128B);
    CUtensorMap tb = make_tmap_2d(W, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (uint64_t)K, (uint64_t)N, (uint64_t)K * 2, BK,
                                  P_BN, CU_TENSOR_MAP_SWIZZLE_128B);
    // (without a residual its map is a further, unused view of W so the kernel signature stays the same)
    CUtensorMap tr = tb, to;
    epilogue_tmaps(ep, M, N, tr, to);
    const int grid = (int)std::min<long long>(tiles, std::max(sms, 1));
    gemm_persistent_kernel<OUT_FP32, ACT><<<grid, PERSISTENT_THREADS, P_SMEM_BYTES, stream>>>(ta, tb, tr, to, p);
    MB_CUDA(cudaGetLastError());
}

int launch_patch_embed(const PatchGather& pg, const __nv_bfloat16* Wg, int N, const Epilogue& ep, cudaStream_t stream) {
    if (pg.n <= 0 || N <= 0) return 0;
    if (pg.S <= 0 || pg.patch <= 0 || pg.S % pg.patch != 0)
        fail(B200_ERR_INTERNAL, "patch gather: image %d is not a multiple of patch %d", pg.S, pg.patch);
    if (N % 32 != 0) fail(B200_ERR_INTERNAL, "patch gather: N = %d must be a multiple of 32", N);
    if (!ep.out_fp32 || ep.act != ACT_NONE) fail(B200_ERR_INTERNAL, "patch gather: fp32 output without activation only");
    check_epilogue(ep);
    configure();
    if (pg.cls != 0 && pg.cls != 1) fail(B200_ERR_INTERNAL, "patch gather: cls = %d must be 0 or 1", pg.cls);
    const int g = pg.S / pg.patch;
    const long long M = (long long)pg.n * (g * g + pg.cls);
    if (M > 0x7fffffffLL) fail(B200_ERR_INVALID_ARG, "patch gather: batch of %d images is too large", pg.n);
    launch_tiles<PROD_PATCH, true, ACT_NONE>(nullptr, 0, Wg, (int)M, N, patch_gather_k(pg.patch), ep, stream, &pg);
    return 1;
}

int launch_conv3x3(const ConvGather& cg, const __nv_bfloat16* Wc, int N, const Epilogue& ep, cudaStream_t stream) {
    if (cg.n <= 0 || N <= 0) return 0;
    if (cg.H <= 0 || cg.W <= 0 || cg.cin < 8 || cg.cin % 8 != 0)
        fail(B200_ERR_INTERNAL, "conv3x3: %d x %d x %d input (cin must be a positive multiple of 8)", cg.H, cg.W, cg.cin);
    if (N % 8 != 0) fail(B200_ERR_INTERNAL, "conv3x3: N = %d must be a multiple of 8", N);
    if (ep.out_fp32 || ep.act != ACT_RELU) fail(B200_ERR_INTERNAL, "conv3x3: bf16 output with ReLU only");
    if ((reinterpret_cast<uintptr_t>(cg.act) & 15) != 0) fail(B200_ERR_INTERNAL, "conv3x3: input not 16-byte aligned");
    check_epilogue(ep);
    configure();
    const long long M = (long long)cg.n * cg.H * cg.W;
    if (M > 0x7fffffffLL) fail(B200_ERR_INVALID_ARG, "conv3x3: batch of %d images is too large", cg.n);
    launch_tiles<PROD_CONV, false, ACT_RELU>(nullptr, 0, Wc, (int)M, N, conv_gather_k(cg.cin), ep, stream, nullptr, &cg);
    return 1;
}

int conv_rows_k(int cin, int k) { return cin == 3 ? 64 : k == 1 ? cin : conv_gather_k(cin); }

int launch_conv(const __nv_bfloat16* x, int n, int H, int W, int cin, int k, const __nv_bfloat16* Wc, int cout,
                const Epilogue& ep, int sms, cudaStream_t stream) {
    if (k == 3 && cin != 3) {
        ConvGather g;
        g.act = x;
        g.n = n;
        g.H = H;
        g.W = W;
        g.cin = cin;
        return launch_conv3x3(g, Wc, cout, ep, stream);
    }
    const int K = conv_rows_k(cin, k);
    return launch(x, K, Wc, n * H * W, cout, K, ep, sms, stream) == KERNEL_NONE ? 0 : 1;
}

void conv_weight_rows(const float* w, int cout, int cin, int k, const double* scale, float* out) {
    const int K = conv_rows_k(cin, k), taps = k * k;
    for (int o = 0; o < cout; ++o) {
        const double s = scale ? scale[o] : 1.0;
        float* row = out + (size_t)o * K;
        for (int j = 0; j < K; ++j) row[j] = 0.f;
        for (int c = 0; c < cin; ++c)
            for (int t = 0; t < taps; ++t)
                row[t * cin + c] = (float)((double)w[((size_t)o * cin + c) * taps + t] * s);
    }
}

int launch(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int M, int N, int K, const Epilogue& ep, int sms,
           cudaStream_t stream) {
    if (M <= 0 || N <= 0) return KERNEL_NONE;
    // TMA needs 16-byte row pitches: K % 8 == 0; a partial last k-block is zero-filled past K in both operands.  The
    // bf16 output's last 64-column box is clipped at N by the TMA store, as at M; the fp32 epilogue keeps whole
    // 32-column boxes.
    if (K <= 0 || K % 8 != 0) fail(B200_ERR_INTERNAL, "gemm: K = %d must be a positive multiple of 8", K);
    if (N % (ep.out_fp32 ? 32 : 8) != 0)
        fail(B200_ERR_INTERNAL, "gemm: N = %d must be a multiple of %d", N, ep.out_fp32 ? 32 : 8);
    if (lda % 8 != 0) fail(B200_ERR_INTERNAL, "gemm: lda = %d must be a multiple of 8", lda);
    check_epilogue(ep);
    configure();
    // The persistent kernel's main loop is faster, but its epilogue is not overlapped: it pays with enough k-blocks per
    // tile (all four ViT-L-14 layer GEMMs, K >= 1024), at least one full wave of tiles, and no half-empty 256-wide
    // column tile (the 384-wide BERTs run slower with one; DESIGN.md §7.5c).
    const long long tiles256 = (long long)((M + BM - 1) / BM) * (N / P_BN);
    // (the persistent kernel has no bf16 residual)
    const bool persistent = K >= 1024 && K % BK == 0 && N % P_BN == 0 && tiles256 >= sms &&
                            (ep.out_fp32 || ep.residual == nullptr);
    dispatch(ep.out_fp32, ep.act, [&](auto out, auto a) {
        constexpr bool OUT_FP32 = decltype(out)::value;
        constexpr int ACT = decltype(a)::value;
        if (persistent)
            launch_persistent<OUT_FP32, ACT>(A, lda, W, M, N, K, ep, sms, stream);
        else
            launch_tiles<PROD_TMA, OUT_FP32, ACT>(A, lda, W, M, N, K, ep, stream);
    });
    return persistent ? KERNEL_PERSISTENT : KERNEL_128x128;
}

}  // namespace gemm
}  // namespace mb
