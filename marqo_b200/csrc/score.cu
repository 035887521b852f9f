// Score + top-k over a GPU-resident fp16 embedding matrix (SURVEY §8 a8).
//
// Reference semantics (executed inside Vespa today, specified by
// src/marqo/core/unstructured_vespa_index/unstructured_vespa_index.py:59-133 and the rank profile in
// src/marqo/core/unstructured_vespa_index/unstructured_vespa_schema.py:225-230,292-294):
//   score(doc) = max over the doc's chunk rows of closeness(q, row);  top-`hits` documents.
//
// Pipeline per group of <= 64 queries:
//   1. scan_kernel<SELECT>  persistent, one CTA per SM.  The corpus is streamed once from HBM by TMA (128-byte
//        swizzle, 16 KB stages) and multiplied against the query block by one wgmma warpgroup (M = 64 queries,
//        N = 128 rows, fp16 x fp16 -> fp32), which stores each tile's scores to shared memory.  Up to dim 1024 the
//        query block is resident in shared memory; above it each stage carries its query k-block (STREAM_Q).  Four
//        epilogue warps read them back (one thread per query) and each keeps a sorted register list of the KP best
//        (key, row, doc) of its query.  Rows of a document that is already listed are dropped only when they are PROVABLY not its best
//        chunk (approximate key more than tol = 2 eps below the listed one).
//   2. merge_kernel  one CTA per query: threshold-filters and sorts the per-CTA lists, RE-SCORES the best M
//        candidates exactly (fp64, fixed summation order — the order oracle/score_oracle.c restates), keeps the
//        best chunk per document, ranks documents under (key desc, doc asc) — all in parallel — and then checks
//        the GUARD:   exact key of the k-th document  >  tau + eps
//        where tau bounds the approximate key of every row that was NOT re-scored (max of the full lists' tails
//        and the best unselected list entry) and eps bounds |approximate - exact| for this query.  When the guard
//        holds no unexamined row can belong to (or reorder) the top-k, so the ids are exact.  Otherwise the query
//        is flagged with a threshold L = (k-th exact key) - eps.
//   3. scan_kernel<COLLECT> + finalize_kernel (only for flagged queries; both exit immediately otherwise):
//        a second pass appends EVERY live row whose approximate key is >= L to a per-query buffer; finalize
//        re-scores all of them exactly and repeats step 2's selection.  Excluded rows have exact key < L + eps
//        <= k-th key, so the result is exact whenever the buffer did not overflow; the host loop grows the buffer /
//        lowers L for the pathological remainder (thousands of exact ties, k larger than the per-CTA lists cover).
// The approximate tensor-core key only SELECTS candidates; ids, rows and scores returned always come from the
// exact pass, and the guard makes "the candidate set contained the true top-k" a checked property, not a hope.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <memory>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "ptx.cuh"
#include "score.cuh"

namespace mb {
namespace score {

constexpr int TILE_N = 128;     // corpus rows per tile (wgmma N)
constexpr int BLOCK_K = 64;     // fp16 elements per 128-byte swizzle row
constexpr int MQ = 64;          // queries per pass (wgmma M)
constexpr int WG_K = 16;
constexpr int KP = 16;          // candidates kept per (CTA, query) list
constexpr int K_SMALL = 10;     // k <= K_SMALL: 64 candidates are re-scored; larger k: up to M_CAP
constexpr int M_SMALL = 64;
constexpr int M_CAP = 384;      // most candidates the merge kernel re-scores exactly
constexpr int K_MERGE_MAX = 160;  // largest k the merge kernel answers itself (needs <= KP * KP list entries)
constexpr int FIN_CAP = 4096;   // most collected rows the device finalize handles (shared memory)
constexpr int MAX_LISTS = 256;  // scan grid clamp (merge_kernel's list-head table)
constexpr int ACC_LD = TILE_N + 4;   // fp32 row pitch of the smem accumulator tile (16-byte rows, conflict-free reads)
constexpr int THREADS = 288;    // warps 0-3 epilogue, warps 4-7 MMA warpgroup, warp 8 TMA
constexpr uint32_t STAGE_BYTES = TILE_N * BLOCK_K * 2;
constexpr uint32_t QCHUNK_BYTES = MQ * BLOCK_K * 2;
constexpr int MAX_DIM = 4096;
constexpr int SMEM_LIMIT = 232448;  // 227 KB
static_assert(K_MERGE_MAX + K_MERGE_MAX / 4 + 16 <= KP * KP, "list-entry threshold trick covers at most KP*KP entries");
static_assert(M_CAP >= K_MERGE_MAX + K_MERGE_MAX / 4 + 16, "M_CAP must cover the candidates needed for K_MERGE_MAX");

enum QueryStatus : int { Q_RESOLVED = 0, Q_NEED = 1 };

// Per-group query state, resident on the device; one D2H copy tells the host everything it needs.
struct QState {
    float eps[MQ];     // bound on |approximate scan key - exact scan key| for any row
    float tol[MQ];     // 2 * eps: same-document chunks closer than this are both kept
    float L[MQ];       // collect threshold (approximate-key domain); +inf = query not flagged
    float qn2[MQ];     // |q|^2 (fp32) — euclidean + score modifiers
    double qn2x[MQ];   // |q|^2 (fp64) — euclidean guard
    double ek[MQ];     // exact scan-domain key of the k-th document (diagnostics / next threshold)
    int status[MQ];
    int cnt[MQ];       // rows appended by the collect pass
    int ndocs[MQ];     // distinct documents the last exact selection saw
    int n_need;        // queries flagged for a(nother) collect pass
    int rounds;        // collect passes run by the no-sync path that still left queries flagged (sticky)
};

struct ScanParams {
    int n_rows;
    int dim;
    int num_tiles;
    int num_stages;
    int nq;
    int metric;
    const int32_t* doc_of_row;  // used when HAS_DOCS
    const float* row_bias;      // used when HAS_BIAS: key = 2 * dot - row_bias[row]  (euclidean: |row|^2)
    const float2* mod;          // used when HAS_MOD: per-document (mult, add); key = mult * closeness + add
    const uint32_t* filter;     // optional document bitset (HAS_DOCS instantiations): bit d clear = document d is excluded
    int64_t filter_docs;        // documents covered by `filter`; documents beyond are excluded
    QState* qs;
    // SELECT mode
    float* out_score;           // [grid][MQ][KP]
    int32_t* out_row;
    int32_t* out_doc;
    // COLLECT mode
    int32_t* cbuf;              // [MQ][ccap] rows
    int ccap;
};

// Two ways to feed the wgmma A operand (the query block):
//   resident (dim <= RESIDENT_MAX_DIM): all dim / 64 query k-blocks are loaded once per CTA and stay in shared memory;
//     they take dim / 64 * 8 KB, so the ring stages get what is left of the 227 KB.
//   streamed: every ring stage carries the query k-block (64 x 64, 8 KB) beside the corpus k-block it multiplies, so
//     shared memory does not grow with dim; the price is 8 KB of L2 -> SM query traffic per 16 KB corpus k-block.
constexpr int RESIDENT_MAX_DIM = 1024;
enum ScanKernel : int { SCAN_RESIDENT_Q = 0, SCAN_STREAMED_Q = 1 };

__host__ __device__ inline size_t scan_smem_bytes(int dim, int stages, bool has_mod = false, bool stream_q = false) {
    const size_t resident_q = stream_q ? 0 : (size_t)(dim / BLOCK_K) * QCHUNK_BYTES;
    const size_t stage_bytes = STAGE_BYTES + (stream_q ? QCHUNK_BYTES : 0);
    return resident_q + (size_t)stages * stage_bytes + (size_t)MQ * ACC_LD * sizeof(float) +
           2 * 4 * TILE_N * sizeof(int32_t) + (has_mod ? 4 * TILE_N * sizeof(float2) : 0) + (2 * 16 + 3) * sizeof(uint64_t) +
           1024 /* alignment slack */;
}

// fp32 closeness of the scan key (dot product, or 2 dot - |row|^2 for euclidean); the exact fp64 form is
// closeness_from_dot() below.  Only evaluated when score modifiers make the ranking non-monotone in the dot product.
__device__ __forceinline__ float closeness_approx(float v, int metric, float qn2) {
    switch (metric) {
        case B200_METRIC_EUCLIDEAN:
            return __fdividef(1.0f, 1.0f + sqrtf(fmaxf(qn2 - v, 0.0f)));
        case B200_METRIC_PRENORMALIZED_ANGULAR:
            return __fdividef(1.0f, 2.0f - v);
        case B200_METRIC_ANGULAR:
            return __fdividef(1.0f, 1.0f + acosf(fminf(1.0f, fmaxf(-1.0f, v))));
        default:
            return v;
    }
}

__device__ __forceinline__ float pick32(const uint32_t (&v)[32], int j) {
    uint32_t r = 0;
#pragma unroll
    for (int t = 0; t < 32; ++t)
        if (t == j) r = v[t];
    return __uint_as_float(r);
}

// Sorted (key desc, arrival order) list insert.  With HAS_DOCS a row whose document is already listed is
//   dropped    when its key is more than tol below the listed one (provably not the document's best chunk),
//   replaces   the listed entry when it is more than tol above it (the listed one is provably not the best),
//   kept too   otherwise (a near-tie: the exact pass decides which chunk represents the document).
template <bool HAS_DOCS>
__device__ __forceinline__ void list_insert(float (&ls)[KP], int (&lr)[KP], int (&ld)[KP], float s, int row, int doc,
                                            float tol) {
    if (HAS_DOCS) {
        int pos = -1;
#pragma unroll
        for (int i = KP - 1; i >= 0; --i)
            if (lr[i] >= 0 && ld[i] == doc) pos = i;   // first (= best) listed entry of this document
        if (pos >= 0) {
            float old = 0.f;
#pragma unroll
            for (int i = 0; i < KP; ++i)
                if (i == pos) old = ls[i];
            if (s < old - tol) return;
            if (s > old + tol) {
#pragma unroll
                for (int i = 0; i < KP - 1; ++i)
                    if (i >= pos) {
                        ls[i] = ls[i + 1];
                        lr[i] = lr[i + 1];
                        ld[i] = ld[i + 1];
                    }
                ls[KP - 1] = -INFINITY;
                lr[KP - 1] = -1;
                ld[KP - 1] = -1;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < KP; ++i) {
        if (s > ls[i]) {
            float ts = ls[i];
            int tr = lr[i], td = ld[i];
            ls[i] = s;
            lr[i] = row;
            ld[i] = doc;
            s = ts;
            row = tr;
            doc = td;
        }
    }
}

// STREAM_Q: the query k-block travels in each ring stage (at byte STAGE_BYTES of the stage) instead of being resident.
template <bool HAS_DOCS, bool HAS_BIAS, bool HAS_MOD, bool COLLECT, bool STREAM_Q>
__global__ void __launch_bounds__(THREADS, 1)
scan_kernel(const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_q, ScanParams p) {
    if (COLLECT) {
        // the fallback pass is always enqueued by the asynchronous entry point; nothing flagged -> nothing to do
        if (*reinterpret_cast<volatile int*>(&p.qs->n_need) == 0) return;
    }
    constexpr uint32_t RING_BYTES = STAGE_BYTES + (STREAM_Q ? QCHUNK_BYTES : 0);   // bytes per ring stage
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int kblocks = p.dim / BLOCK_K;
    const int S = p.num_stages;
    uint8_t* smem_q = smem;
    uint8_t* smem_c = smem_q + (STREAM_Q ? 0 : (size_t)kblocks * QCHUNK_BYTES);
    float* smem_acc = reinterpret_cast<float*>(smem_c + (size_t)S * RING_BYTES);
    int32_t* smem_docs = reinterpret_cast<int32_t*>(smem_acc + MQ * ACC_LD);
    float* smem_bias = reinterpret_cast<float*>(smem_docs + 4 * TILE_N);
    float2* smem_mod = reinterpret_cast<float2*>(smem_bias + 4 * TILE_N);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_mod + (HAS_MOD ? 4 * TILE_N : 0));
    uint64_t* empty = full + 16;
    uint64_t* afull = empty + 16;
    uint64_t* aempty = afull + 1;
    uint64_t* qfull = aempty + 1;

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const int lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmap_c);
        ptx::prefetch_tmap(&tmap_q);
        for (int i = 0; i < S; ++i) {
            ptx::mbar_init(&full[i], 1);
            ptx::mbar_init(&empty[i], 4);   // one arrive per MMA warp
        }
        ptx::mbar_init(afull, 128);         // every MMA thread has stored its accumulators
        ptx::mbar_init(aempty, 4);          // every epilogue warp has read the tile
        ptx::mbar_init(qfull, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ------------------------------------------------------------ TMA producer
        if (lane == 0) {
            if constexpr (!STREAM_Q) {
                ptx::mbar_arrive_expect_tx(qfull, kblocks * QCHUNK_BYTES);
                for (int kb = 0; kb < kblocks; ++kb)
                    ptx::tma_load_2d(smem_q + (size_t)kb * QCHUNK_BYTES, &tmap_q, qfull, kb * BLOCK_K, 0, ptx::kEvictLast);
            }
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
                for (int kb = 0; kb < kblocks; ++kb) {
                    ptx::mbar_wait(&empty[stage], phase ^ 1);
                    ptx::mbar_arrive_expect_tx(&full[stage], RING_BYTES);
                    ptx::tma_load_2d(smem_c + (size_t)stage * RING_BYTES, &tmap_c, &full[stage], kb * BLOCK_K,
                                     tile * TILE_N, ptx::kEvictFirst);
                    if constexpr (STREAM_Q)   // the query block is re-read by every CTA for every tile: keep it in L2
                        ptx::tma_load_2d(smem_c + (size_t)stage * RING_BYTES + STAGE_BYTES, &tmap_q, &full[stage],
                                         kb * BLOCK_K, 0, ptx::kEvictLast);
                    if (++stage == S) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else if (warp >= 4) {
        // ------------------------------------------------------------ MMA warpgroup: S = Q C^T for one tile (64 x 128)
        if constexpr (!STREAM_Q) ptx::mbar_wait(qfull, 0);
        const int r0 = (warp - 4) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
        int stage = 0;
        uint32_t phase = 0, acc_phase = 0;
        float acc[TILE_N / 2];
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
            for (int kb = 0; kb < kblocks; ++kb) {
                ptx::mbar_wait(&full[stage], phase);
                const uint32_t a_base = ptx::smem_u32(STREAM_Q ? smem_c + (size_t)stage * RING_BYTES + STAGE_BYTES
                                                               : smem_q + (size_t)kb * QCHUNK_BYTES);
                const uint32_t b_base = ptx::smem_u32(smem_c + (size_t)stage * RING_BYTES);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < BLOCK_K / WG_K; ++k)
                    ptx::wgmma_m64n128k16_f16(acc, ptx::make_desc_k_sw128(a_base + k * WG_K * 2),
                                              ptx::make_desc_k_sw128(b_base + k * WG_K * 2), (kb | k) != 0 ? 1u : 0u);
                ptx::wgmma_commit();
                ptx::wgmma_wait<0>();
                __syncwarp();
                if (lane == 0) ptx::mbar_arrive(&empty[stage]);
                if (++stage == S) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            // hand the tile to the epilogue warps through smem (row = query, ACC_LD-float rows)
            ptx::mbar_wait(aempty, acc_phase ^ 1);
#pragma unroll
            for (int i = 0; i < TILE_N / 8; ++i) {
                *reinterpret_cast<float2*>(smem_acc + r0 * ACC_LD + 8 * i + c0) = make_float2(acc[4 * i], acc[4 * i + 1]);
                *reinterpret_cast<float2*>(smem_acc + (r0 + 8) * ACC_LD + 8 * i + c0) =
                    make_float2(acc[4 * i + 2], acc[4 * i + 3]);
            }
            ptx::mbar_arrive(afull);
            acc_phase ^= 1;
        }
    } else {
        // ------------------------------------------------------------ epilogue: per-query running top-KP / collect
        const int q = warp * 16 + lane;  // lanes 0-15 of warp w own queries 16 w .. 16 w + 15
        const bool active = lane < 16 && q < p.nq;
        int32_t* my_docs = smem_docs + warp * TILE_N;
        float* my_bias = smem_bias + warp * TILE_N;
        float2* my_mod = smem_mod + (HAS_MOD ? warp * TILE_N : 0);
        const float* my_acc = smem_acc + (lane < 16 ? q : 0) * ACC_LD;
        const float my_qn2 = (HAS_MOD && active) ? p.qs->qn2[q] : 0.f;
        const float tol = (HAS_DOCS && active && !COLLECT) ? p.qs->tol[q] : 0.f;
        float ls[KP];
        int lr[KP], ld[KP];
#pragma unroll
        for (int i = 0; i < KP; ++i) {
            ls[i] = -INFINITY;
            lr[i] = -1;
            ld[i] = -1;
        }
        // SELECT: a row qualifies when key > thr (the list's tail).  COLLECT: when key >= thr (= L[q]; +inf when
        // the query is not flagged).
        float thr = -INFINITY;
        if (COLLECT) thr = active ? p.qs->L[q] : INFINITY;
        const uint32_t* filt = HAS_DOCS ? p.filter : nullptr;
        uint32_t acc_phase = 0;
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
            const int row0 = tile * TILE_N;
            if (HAS_DOCS || HAS_BIAS || HAS_MOD) {
                __syncwarp();
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    int r = row0 + t * 32 + lane;
                    int d = r;
                    if (HAS_DOCS) {
                        d = r < p.n_rows ? __ldg(p.doc_of_row + r) : -1;
                        if (filt != nullptr && d >= 0) {
                            const bool keep = d < p.filter_docs && ((__ldg(filt + (d >> 5)) >> (d & 31)) & 1u);
                            if (!keep) d = -1;   // a filtered-out document looks like a deleted row
                        }
                        my_docs[t * 32 + lane] = d;
                    }
                    if (HAS_BIAS) my_bias[t * 32 + lane] = r < p.n_rows ? __ldg(p.row_bias + r) : 0.f;
                    if (HAS_MOD) my_mod[t * 32 + lane] = (r < p.n_rows && d >= 0) ? __ldg(p.mod + d) : make_float2(0.f, 0.f);
                }
                __syncwarp();
            }
            ptx::mbar_wait(afull, acc_phase);
            const int valid = min(TILE_N, p.n_rows - row0);
#pragma unroll 1
            for (int c = 0; c < TILE_N / 32; ++c) {
                uint32_t v[32];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float4 f4 = *reinterpret_cast<const float4*>(my_acc + c * 32 + 4 * j);
                    v[4 * j] = __float_as_uint(f4.x);
                    v[4 * j + 1] = __float_as_uint(f4.y);
                    v[4 * j + 2] = __float_as_uint(f4.z);
                    v[4 * j + 3] = __float_as_uint(f4.w);
                }
                if (c == TILE_N / 32 - 1) {
                    // the whole row is in registers: hand the buffer back to the MMA warpgroup
                    __syncwarp();
                    if (lane == 0) ptx::mbar_arrive(aempty);
                }
                if (active) {
                    if (HAS_BIAS) {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            v[j] = __float_as_uint(fmaf(2.0f, __uint_as_float(v[j]), -my_bias[c * 32 + j]));
                    }
                    if (HAS_MOD) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const float2 ma = my_mod[c * 32 + j];
                            v[j] = __float_as_uint(fmaf(ma.x, closeness_approx(__uint_as_float(v[j]), p.metric, my_qn2), ma.y));
                        }
                    }
                    uint32_t mask = 0;
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        const float f = __uint_as_float(v[j]);
                        mask |= (COLLECT ? (f >= thr) : (f > thr)) ? (1u << j) : 0u;
                    }
                    const int nvalid = valid - c * 32;
                    if (nvalid < 32) mask &= nvalid <= 0 ? 0u : ((1u << nvalid) - 1u);
                    while (mask) {
                        const int j = __ffs(mask) - 1;
                        mask &= mask - 1;
                        const float s = pick32(v, j);
                        const int row = row0 + c * 32 + j;
                        if (!COLLECT && !(s > thr)) continue;
                        int doc = row;
                        if (HAS_DOCS) {
                            doc = my_docs[c * 32 + j];
                            if (doc < 0) continue;  // tombstoned or filtered-out row
                        }
                        if (COLLECT) {
                            const int slot = atomicAdd(&p.qs->cnt[q], 1);
                            if (slot < p.ccap) p.cbuf[(size_t)q * p.ccap + slot] = row;
                        } else {
                            list_insert<HAS_DOCS>(ls, lr, ld, s, row, doc, tol);
                            thr = ls[KP - 1];
                        }
                    }
                }
            }
            acc_phase ^= 1;
        }
        if (!COLLECT && lane < 16) {
            const size_t base = ((size_t)blockIdx.x * MQ + q) * KP;
#pragma unroll
            for (int i = 0; i < KP; ++i) {
                p.out_score[base + i] = ls[i];
                p.out_row[base + i] = lr[i];
                p.out_doc[base + i] = ld[i];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Exact selection shared by merge_kernel (candidates from the per-CTA lists) and finalize_kernel (rows from the
// collect pass).
struct ExactParams {
    int nq;
    int k;
    int dim;
    int metric;
    int doc_offset;        // added to every returned document number (global numbering of a row-sharded corpus)
    const __half* qh;      // [MQ, dim] fp16 queries as scanned
    const __half* corpus;  // [n_rows, dim]
    const int32_t* doc_of_row;
    const double2* mod64;  // optional score modifiers: per-document (mult, add) in fp64; key = mult * closeness + add
    QState* qs;
    int32_t* out_doc;      // [nq, k]
    int32_t* out_row;
    double* out_score;
};

// `dot` is the exact dot product of the re-score pass, or minus the squared distance (euclidean).  Device code
// takes CUDA's sqrt / acos, host code (host_finalize) libm's.
__host__ __device__ __forceinline__ double closeness_from_dot(double dot, int metric) {
    switch (metric) {
        case B200_METRIC_EUCLIDEAN:
            return 1.0 / (1.0 + sqrt(fmax(-dot, 0.0)));
        case B200_METRIC_PRENORMALIZED_ANGULAR:
            return 1.0 / (1.0 + (1.0 - dot));
        case B200_METRIC_ANGULAR: {
            double c = fmin(1.0, fmax(-1.0, dot));
            return 1.0 / (1.0 + acos(c));
        }
        default:
            return dot;
    }
}

// Exact ordering key of a re-scored row: its dot product, or with score modifiers the modified score
// mult * closeness + add of its document (separate multiply and add, no fma, as oracle/score_oracle.c computes it).
// `doc` is read only with modifiers.
__device__ __forceinline__ double exact_key(const ExactParams& p, double dot, const int32_t& doc) {
    if (!p.mod64) return dot;
    const double2 ma = p.mod64[doc];
    return __dadd_rn(__dmul_rn(ma.x, closeness_from_dot(dot, p.metric)), ma.y);
}

// Score returned for an exact key: the modified score itself, or the closeness of the dot product.
__host__ __device__ __forceinline__ double key_score(double key, int metric, bool modified) {
    return modified ? key : closeness_from_dot(key, metric);
}

// Scan-domain key (what the scan's approximate key approximates) of an exact key: the modified score, the dot
// product, or for euclidean -|q - e|^2 + |q|^2 = 2 q.e - |e|^2.  `qn2` (|q|^2) is read only for euclidean.
__host__ __device__ __forceinline__ double scan_domain_key(double key, int metric, bool modified, const double& qn2) {
    return modified ? key : (metric == B200_METRIC_EUCLIDEAN ? key + qn2 : key);
}

// Largest float <= x.
__host__ __device__ __forceinline__ float float_rd(double x) {
#ifdef __CUDA_ARCH__
    return __double2float_rd(x);
#else
    const float f = (float)x;
    return (double)f > x ? std::nextafterf(f, -INFINITY) : f;
#endif
}

// Records query q's exact selection (nd distinct documents, k-th scan-domain key ek) and settles the query: either
// resolved, or flagged for another collect pass with threshold next_L() (only evaluated then).  Returns true when
// the query needs that pass; the caller counts it in n_need.
template <class NextL>
__host__ __device__ __forceinline__ bool settle(QState* qs, int q, int nd, double ek, bool resolved, NextL next_L) {
    qs->ndocs[q] = nd;
    qs->ek[q] = ek;
    qs->cnt[q] = 0;
    if (resolved) {
        qs->status[q] = Q_RESOLVED;
        qs->L[q] = INFINITY;
    } else {
        qs->L[q] = next_L();
        qs->status[q] = Q_NEED;
    }
    return !resolved;
}

// Settles a query after an exact selection over every row the collect pass found at threshold L (finalize_kernel
// and host_finalize).  A row that was not collected has approximate key < L, so exact key < L + eps: the top-k is
// exact once the k-th exact key reaches L + eps, or when L = -inf collected every live row.  Otherwise the next
// threshold is ek - eps rounded down (every row whose exact key can reach ek has approximate key >= it), or, with
// fewer than k documents above L, L lowered by max(8 eps, 5 % of |L|); -inf (collect everything) when that is not
// below L.
__host__ __device__ __forceinline__ bool settle_collected(QState* qs, int q, int k, int nd, double ek) {
    const float L = qs->L[q];
    const float eps = qs->eps[q];
    const bool resolved = (L == -INFINITY) || (nd >= k && ek >= (double)L + (double)eps);
    return settle(qs, q, nd, ek, resolved, [&] {
        float nl;
        if (nd >= k) nl = float_rd(ek - (double)eps);
        else nl = L - fmaxf(8.0f * eps, 0.05f * fabsf(L));
        if (!(nl < L)) nl = -INFINITY;
        return nl;
    });
}

// Exact fp64 dot product (or minus squared distance) of query `qv` and corpus row `cv`, computed by one warp.
// Fixed order, restated by oracle/score_oracle.c: lane l accumulates elements i = 256 j + 8 l + t (j ascending, then
// t = 0..7), lanes are combined by the xor butterfly 16, 8, 4, 2, 1.  Every product of two fp16 values is exact in
// fp64, so fused and unfused multiply-add give the same bits; the euclidean form uses explicit unfused ops.
__device__ __forceinline__ double warp_exact_dot(const __half* __restrict__ qv, const __half* __restrict__ cv, int dim,
                                                 int metric, int lane) {
    double part = 0.0;
    for (int base = 8 * lane; base < dim; base += 256) {
        const uint4 qa = *reinterpret_cast<const uint4*>(qv + base);
        const uint4 ca = __ldg(reinterpret_cast<const uint4*>(cv + base));
        const __half2* qh2 = reinterpret_cast<const __half2*>(&qa);
        const __half2* ch2 = reinterpret_cast<const __half2*>(&ca);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 qf = __half22float2(qh2[t]);
            const float2 cf = __half22float2(ch2[t]);
            if (metric == B200_METRIC_EUCLIDEAN) {
                const double d0 = (double)qf.x - (double)cf.x;   // exact in fp64
                const double d1 = (double)qf.y - (double)cf.y;
                part = __dsub_rn(part, __dmul_rn(d0, d0));
                part = __dsub_rn(part, __dmul_rn(d1, d1));
            } else {
                part = __dadd_rn(part, __dmul_rn((double)qf.x, (double)cf.x));
                part = __dadd_rn(part, __dmul_rn((double)qf.y, (double)cf.y));
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part = __dadd_rn(part, __shfl_xor_sync(0xffffffffu, part, o));
    return part;
}

// Block-wide: re-score entries [0, n) (rows in s_row) exactly, keep each document's best chunk (dot desc, row asc),
// rank the documents by (key desc, doc asc) and write the best k.  Returns (through smem) the number of distinct
// documents and the exact scan-domain key of the k-th one.
//   scan-domain key = what the scan's approximate key approximates: dot | dot + |q|^2 (euclidean: 2 q.e - |e|^2) |
//   the modified score.
template <int NTHREADS>
__device__ void exact_select(const ExactParams& p, int q, int n, const int32_t* s_row, int32_t* s_doc, double* x_dot,
                             double* x_key, uint8_t* x_rep, int* s_ndocs, double* s_ek) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const __half* qv = p.qh + (size_t)q * p.dim;
    for (int c = warp; c < n; c += NTHREADS / 32) {
        const int row = s_row[c];
        const double tot = warp_exact_dot(qv, p.corpus + (size_t)row * p.dim, p.dim, p.metric, lane);
        if (lane == 0) {
            x_dot[c] = tot;
            x_key[c] = exact_key(p, tot, s_doc[c]);
        }
    }
    if (threadIdx.x == 0) {
        *s_ndocs = 0;
        *s_ek = -INFINITY;
    }
    __syncthreads();
    // best chunk per document
    for (int i = threadIdx.x; i < n; i += NTHREADS) {
        const int d = s_doc[i], r = s_row[i];
        const double v = x_dot[i];
        bool rep = true;
        for (int j = 0; j < n; ++j)
            rep &= !(s_doc[j] == d && (x_dot[j] > v || (x_dot[j] == v && s_row[j] < r)));
        x_rep[i] = rep ? 1 : 0;
        if (rep) atomicAdd(s_ndocs, 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += NTHREADS) {
        if (!x_rep[i]) continue;
        const int d = s_doc[i];
        const double v = x_key[i];
        int rank = 0;
        for (int j = 0; j < n; ++j) rank += (x_rep[j] && (x_key[j] > v || (x_key[j] == v && s_doc[j] < d))) ? 1 : 0;
        if (rank < p.k) {
            const size_t o = (size_t)q * p.k + rank;
            p.out_doc[o] = d + p.doc_offset;
            p.out_row[o] = s_row[i];
            p.out_score[o] = key_score(v, p.metric, p.mod64);
            if (rank == p.k - 1) *s_ek = scan_domain_key(v, p.metric, p.mod64, p.qs->qn2x[q]);
        }
    }
    __syncthreads();
    const int nd = *s_ndocs;
    for (int i = nd + threadIdx.x; i < p.k; i += NTHREADS) {
        const size_t o = (size_t)q * p.k + i;
        p.out_doc[o] = -1;
        p.out_row[o] = -1;
        p.out_score[o] = -INFINITY;
    }
}

// monotone float <-> uint32 map (for shared-memory atomicMax / atomicMin on scores of either sign)
__device__ __forceinline__ uint32_t flt_key(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_flt(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct MergeParams {
    int num_lists;  // scan grid size
    int sort_n;     // power of two >= num_lists * KP
    int l_only;     // k > K_MERGE_MAX: only choose the collect threshold L (the collect pass answers)
    const float* in_score;
    const int32_t* in_row;
    const int32_t* in_doc;
    ExactParams ex;
};

__device__ __forceinline__ bool approx_before(float sa, int ra, float sb, int rb) {
    return sa > sb || (sa == sb && ra < rb);
}

constexpr int MERGE_THREADS = 256;

__global__ void __launch_bounds__(MERGE_THREADS) merge_kernel(MergeParams p) {
    extern __shared__ uint8_t msmem[];
    float* s_score = reinterpret_cast<float*>(msmem);
    int32_t* s_row = reinterpret_cast<int32_t*>(s_score + p.sort_n);
    int32_t* s_doc = s_row + p.sort_n;
    __shared__ double x_dot[M_CAP], x_key[M_CAP];
    __shared__ uint8_t x_rep[M_CAP];
    __shared__ float s_head[MAX_LISTS];
    __shared__ float s_thr;
    __shared__ uint32_t s_tail_max, s_below_max, s_union_min;
    __shared__ int s_count, s_ndocs;
    __shared__ double s_ek;

    const int q = blockIdx.x;
    const int k = p.ex.k;
    QState* qs = p.ex.qs;
    const int total = p.num_lists * KP;
    // candidates wanted from the lists: enough that the k-th exact key clears the best unselected entry
    const int need = p.l_only ? INT_MAX : (k <= K_SMALL ? KP : k + k / 4 + 16);
    const int e_sel = p.l_only ? 0 : (need + KP - 1) / KP - 1;   // <= KP - 1 by the static_asserts
    if (threadIdx.x == 0) {
        s_thr = -INFINITY;
        s_tail_max = flt_key(-INFINITY);
        s_below_max = flt_key(-INFINITY);
        s_union_min = flt_key(INFINITY);
        s_count = 0;
    }
    __syncthreads();
    // Every list is sorted, so the KP-th largest of the lists' e_sel-th entries is a lower bound of the global
    // KP*(e_sel+1)-th best key: only candidates >= that bound are wanted.  Shrinks the sort from ~2.4k keys to ~need.
    for (int l = threadIdx.x; l < p.num_lists; l += blockDim.x) {
        const size_t src = ((size_t)l * MQ + q) * KP;
        s_head[l] = p.in_row[src + e_sel] >= 0 ? p.in_score[src + e_sel] : -INFINITY;
        // a FULL list may have rejected rows: its tail bounds their keys
        if (p.in_row[src + KP - 1] >= 0) atomicMax(&s_tail_max, flt_key(p.in_score[src + KP - 1]));
    }
    __syncthreads();
    if (!p.l_only && p.num_lists >= KP) {
        for (int l = threadIdx.x; l < p.num_lists; l += blockDim.x) {
            const float h = s_head[l];
            int rank = 0;
            for (int j = 0; j < p.num_lists; ++j) rank += (s_head[j] > h) || (s_head[j] == h && j < l);
            if (rank == KP - 1) s_thr = h;
        }
    }
    __syncthreads();
    const float thr = s_thr;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        const int list = i / KP, e = i % KP;
        const size_t src = ((size_t)list * MQ + q) * KP + e;
        const int rr = p.in_row[src];
        if (rr < 0) continue;
        const float sc = p.in_score[src];
        atomicMin(&s_union_min, flt_key(sc));
        if (sc >= thr) {
            const int slot = atomicAdd(&s_count, 1);
            s_score[slot] = sc;
            s_row[slot] = rr;
            s_doc[slot] = p.in_doc[src];
        } else {
            atomicMax(&s_below_max, flt_key(sc));
        }
    }
    __syncthreads();
    const int count = s_count;
    int n2 = 32;
    while (n2 < count) n2 <<= 1;
    for (int i = count + threadIdx.x; i < n2; i += blockDim.x) {
        s_score[i] = -INFINITY;
        s_row[i] = INT_MAX;
        s_doc[i] = -1;
    }
    __syncthreads();
    // bitonic sort, order: (key desc, row asc) — a total order, so the result does not depend on slot order
    for (int size = 2; size <= n2; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = threadIdx.x; i < n2 / 2; i += blockDim.x) {
                const int lo = 2 * i - (i & (stride - 1));
                const int hi = lo + stride;
                const bool up = (lo & size) == 0;
                const float sa = s_score[lo], sb = s_score[hi];
                const int ra = s_row[lo], rb = s_row[hi];
                const bool wrong = up ? approx_before(sb, rb, sa, ra) : approx_before(sa, ra, sb, rb);
                if (wrong) {
                    s_score[lo] = sb;
                    s_score[hi] = sa;
                    s_row[lo] = rb;
                    s_row[hi] = ra;
                    const int da = s_doc[lo];
                    s_doc[lo] = s_doc[hi];
                    s_doc[hi] = da;
                }
            }
            __syncthreads();
        }
    }
    const float eps = qs->eps[q];
    if (p.l_only) {
        // k beyond the merge kernel's reach: collect every row at least as good as the (k + slack)-th list entry
        if (threadIdx.x == 0) {
            const int want = k + k / 8 + 16;
            float L = -INFINITY;   // fewer entries than wanted and no list is full: the lists ARE the corpus
            if (count >= want) L = s_score[want - 1];
            else if (key_flt(s_tail_max) > -INFINITY) L = key_flt(s_union_min);
            qs->L[q] = L;
            qs->cnt[q] = 0;
            qs->status[q] = Q_NEED;
            atomicAdd(&qs->n_need, 1);
        }
        return;
    }
    const int mcap = k <= K_SMALL ? M_SMALL : M_CAP;
    const int M = min(count, mcap);
    exact_select<MERGE_THREADS>(p.ex, q, M, s_row, s_doc, x_dot, x_key, x_rep, &s_ndocs, &s_ek);
    __syncthreads();
    if (threadIdx.x == 0) {
        // tau: upper bound of the approximate key of every live row that was not re-scored
        const float tau_m = count > M ? s_score[M] : key_flt(s_below_max);
        const float tau = fmaxf(key_flt(s_tail_max), tau_m);
        const int nd = s_ndocs;
        const bool resolved = nd >= k ? (s_ek > (double)tau + (double)eps) : (tau == -INFINITY);
        const bool need = settle(qs, q, nd, s_ek, resolved, [&] {
            // every row whose exact key can reach the k-th one has approximate key >= ek - eps; with fewer than k
            // documents in hand start from the weakest list entry
            return nd >= k ? float_rd(s_ek - (double)eps) : key_flt(s_union_min);
        });
        if (need) atomicAdd(&qs->n_need, 1);
    }
}

// One CTA per flagged query: exact selection over the rows appended by the collect pass.
constexpr int FIN_THREADS = 512;
struct FinalizeParams {
    const int32_t* cbuf;
    int ccap;
    int64_t live_bound;   // n_rows: a collect pass with L = -inf saw every live row
    ExactParams ex;
};

__host__ __device__ inline size_t finalize_smem_bytes(int n) { return (size_t)n * (4 + 4 + 8 + 8 + 1) + 64; }

__global__ void __launch_bounds__(FIN_THREADS) finalize_kernel(FinalizeParams p) {
    extern __shared__ __align__(16) uint8_t fsmem[];
    QState* qs = p.ex.qs;
    const int q = blockIdx.x;
    if (qs->status[q] != Q_NEED) return;
    const int cnt = qs->cnt[q];
    const int k = p.ex.k;
    __shared__ int s_ndocs;
    __shared__ double s_ek;
    if (cnt > p.ccap || cnt > FIN_CAP) {   // overflow: the host grows the buffer / finalizes on the host
        if (threadIdx.x == 0) atomicAdd(&qs->n_need, 1);
        return;
    }
    double* x_dot = reinterpret_cast<double*>(fsmem);
    double* x_key = x_dot + cnt;
    int32_t* s_row = reinterpret_cast<int32_t*>(x_key + cnt);
    int32_t* s_doc = s_row + cnt;
    uint8_t* x_rep = reinterpret_cast<uint8_t*>(s_doc + cnt);
    for (int i = threadIdx.x; i < cnt; i += FIN_THREADS) {
        const int r = p.cbuf[(size_t)q * p.ccap + i];
        s_row[i] = r;
        s_doc[i] = p.ex.doc_of_row[r];
    }
    __syncthreads();
    exact_select<FIN_THREADS>(p.ex, q, cnt, s_row, s_doc, x_dot, x_key, x_rep, &s_ndocs, &s_ek);
    __syncthreads();
    if (threadIdx.x == 0 && settle_collected(qs, q, k, s_ndocs, s_ek)) atomicAdd(&qs->n_need, 1);
}

// Host-finalize support: exact dot and key of every collected row of one query (warp per row).
__global__ void exact_keys_kernel(ExactParams p, int q, const int32_t* rows, int n, double* out_dot, double* out_key,
                                  int32_t* out_doc) {
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    const int row = rows[i];
    const double tot = warp_exact_dot(p.qh + (size_t)q * p.dim, p.corpus + (size_t)row * p.dim, p.dim, p.metric, lane);
    if (lane == 0) {
        const int d = p.doc_of_row[row];
        const double key = exact_key(p, tot, d);
        out_dot[i] = tot;
        out_key[i] = key;
        out_doc[i] = d;
    }
}

// Per-query error bound of the approximate scan key (warp per query).  fp16 x fp16 products are exact in fp32; the
// tensor core adds them (16 per instruction, dim / 16 instructions) with at most one truncation per addend, so
//   |approx dot - exact dot| <= dim * 2^-23 * sum|q_i e_i| <= dim * 2^-23 * |q| |e|.
// The bound used is twice that (c = dim * 2^-22) with |e| <= sqrt(max_n2), the largest stored row norm.
// Measured on the H100 (tests/test_score_bound_gpu.py): wgmma adds each group of four products exactly and truncates
// the sum once, so the worst error seen is a quarter of the per-addend model, 1/8 of the dot-product eps.
__global__ void query_prep_kernel(const __half* __restrict__ qh, int dim, int metric, int has_mod,
                                  const float* __restrict__ max_n2, const double* __restrict__ mod_max, QState* qs) {
    const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= MQ) return;
    double n2 = 0.0;
    for (int i = lane; i < dim; i += 32) {
        const double f = (double)__half2float(qh[(size_t)q * dim + i]);
        n2 += f * f;
    }
    for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
    if (lane != 0) return;
    const float qn = sqrtf((float)n2) * 1.001f;
    const float R = sqrtf(*max_n2) * 1.001f;
    const float c = (float)dim * 2.384185791015625e-07f;   // dim * 2^-22
    float eps = c * qn * R;                                // dot-product domain
    if (metric == B200_METRIC_EUCLIDEAN)                   // key = fma(2, dot, -n2_fp32[row])
        eps = 2.0f * eps + 0.5f * c * R * R + 4.76837158203125e-07f * (2.0f * qn * R + R * R);
    if (has_mod) {
        // key = fma(mult32, closeness32(v), add32); closeness error from the error eps of v:
        float ec;
        switch (metric) {
            case B200_METRIC_PRENORMALIZED_ANGULAR: {   // 1/(2 - v): Lipschitz 1/(2 - vmax)^2
                const float room = 2.0f - qn * R - eps;
                ec = room > 0.05f ? eps / (room * room) : INFINITY;
                break;
            }
            case B200_METRIC_ANGULAR:                     // |acos a - acos b| <= 2 sqrt|a - b|, |d closeness / d theta| <= 1
                ec = 2.0f * sqrtf(eps);
                break;
            case B200_METRIC_EUCLIDEAN:                   // |sqrt a - sqrt b| <= sqrt|a - b|
                ec = sqrtf(eps + 4.76837158203125e-07f * qn * qn);
                break;
            default:
                ec = eps;
        }
        const float mmax = (float)mod_max[0] * 1.001f, amax = (float)mod_max[1] * 1.001f;
        eps = mmax * (ec + 1e-6f) + (mmax + amax) * 4.76837158203125e-07f;
    }
    eps += 1e-30f;
    qs->eps[q] = eps;
    qs->tol[q] = 2.0f * eps;
    qs->L[q] = INFINITY;
    qs->qn2[q] = (float)n2;
    qs->qn2x[q] = n2;
    qs->status[q] = Q_RESOLVED;
    qs->cnt[q] = 0;
    qs->ndocs[q] = 0;
    qs->ek[q] = 0.0;
    if (q == 0) qs->n_need = 0;
}

__global__ void reset_need_kernel(QState* qs) { qs->n_need = 0; }
__global__ void note_unresolved_kernel(QState* qs) {
    if (qs->n_need > 0) qs->rounds += 1;
}

// ------------------------------------------------------------------------------------------------
// fp32 -> fp16 row conversion (optionally L2-normalising first, for the angular metric).
// `flags`: bit 0 is set when a value is not finite or does not fit fp16 (|x| > 65504 after normalisation);
// `max_n2` accumulates the largest squared norm of the STORED rows (the error bound of the scan needs it).
__global__ void convert_rows_kernel(const float* __restrict__ src, __half* __restrict__ dst, int64_t rows, int dim,
                                    int64_t dst_rows_total, int normalize, float* __restrict__ n2_out,
                                    float* __restrict__ max_n2, int* __restrict__ flags) {
    // one warp per row; rows in [rows, dst_rows_total) are zero-filled (query padding)
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= dst_rows_total) return;
    __half* d = dst + row * dim;
    if (row >= rows) {
        for (int i = lane; i < dim; i += 32) d[i] = __float2half_rn(0.f);
        return;
    }
    const float* s = src + row * dim;
    float scale = 1.f;
    if (normalize) {
        float ss = 0.f;
        for (int i = lane; i < dim; i += 32) ss = __fmaf_rn(s[i], s[i], ss);
        for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        scale = ss > 0.f ? 1.0f / sqrtf(ss) : 0.f;
    }
    float n2 = 0.f;
    bool bad = false;
    for (int i = lane; i < dim; i += 32) {
        const float x = s[i] * scale;
        bad |= !(fabsf(x) <= 65504.0f);   // also true for NaN
        const __half hv = __float2half_rn(x);
        d[i] = hv;
        const float f = __half2float(hv);
        n2 = fmaf(f, f, n2);
    }
    for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
    if (__any_sync(0xffffffffu, bad) && lane == 0 && flags) atomicOr(flags, 1);
    if (lane == 0) {
        if (n2_out) n2_out[row] = n2;   // |row|^2 of the STORED (fp16-rounded) values: the euclidean scan's per-row term
        if (max_n2 && n2 == n2 && n2 < INFINITY) atomicMax(reinterpret_cast<int*>(max_n2), __float_as_int(n2));   // n2 >= 0
    }
}

__global__ void row_norms_kernel(const __half* __restrict__ rows, int64_t n, int dim, float* __restrict__ n2_out,
                                 float* __restrict__ max_n2) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    float n2 = 0.f;
    for (int i = lane; i < dim; i += 32) {
        const float f = __half2float(rows[row * dim + i]);
        n2 = fmaf(f, f, n2);
    }
    for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
    if (lane == 0) {
        if (n2_out) n2_out[row] = n2;
        if (n2 == n2 && n2 < INFINITY) atomicMax(reinterpret_cast<int*>(max_n2), __float_as_int(n2));
    }
}

__global__ void iota_kernel(int32_t* dst, int64_t n, int32_t start) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = start + (int32_t)i;
}

__global__ void tombstone_kernel(int32_t* doc_of_row, int64_t n, int32_t doc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && doc_of_row[i] == doc) doc_of_row[i] = -1;
}

__global__ void tombstone_rows_kernel(int32_t* doc_of_row, const int32_t* rows, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) doc_of_row[rows[i]] = -1;
}

// compaction: copy live rows to their new positions (one warp per OLD row; new_of_old[row] < 0 = dead)
__global__ void compact_rows_kernel(const __half* __restrict__ src, __half* __restrict__ dst,
                                    const int32_t* __restrict__ src_doc, int32_t* __restrict__ dst_doc,
                                    const float* __restrict__ src_n2, float* __restrict__ dst_n2,
                                    const int32_t* __restrict__ new_of_old, int64_t n, int dim) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    const int32_t to = new_of_old[row];
    if (to < 0) return;
    const uint4* s = reinterpret_cast<const uint4*>(src + row * dim);
    uint4* d = reinterpret_cast<uint4*>(dst + (int64_t)to * dim);
    for (int i = lane; i < dim / 8; i += 32) d[i] = s[i];
    if (lane == 0) {
        dst_doc[to] = src_doc[row];
        if (src_n2) dst_n2[to] = src_n2[row];
    }
}

// Score modifiers (reference: the rank-profile function `modify`, unstructured_vespa_schema.py:266-271):
//   mult = count(mult_w * attr) == 0 ? 1 : prod(mult_w * attr);   add = sum(add_w * attr)
// over the attribute cells a document HAS (NaN = missing cell of the sparse tensor<double>(p{})), in the order the
// caller lists the columns.  Written in fp64 for the exact merge and in fp32 for the scan.
constexpr int MAX_MOD_TERMS = 16;
struct ModifierParams {
    int n_docs;
    int attr_cap;
    int n_mult, n_add;
    const double* mult_col[MAX_MOD_TERMS];
    const double* add_col[MAX_MOD_TERMS];
    double mult_w[MAX_MOD_TERMS];
    double add_w[MAX_MOD_TERMS];
    double2* out64;
    float2* out32;
    int* negative_flag;
    double* mod_max;   // [2]: max |mult|, max |add| over the documents (error bound of the modified scan key)
};

__global__ void modifier_kernel(ModifierParams p) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= p.n_docs) return;
    double m = 1.0, a = 0.0;
    int cnt = 0;
    for (int i = 0; i < p.n_mult; ++i) {
        const double v = (p.mult_col[i] && d < p.attr_cap) ? p.mult_col[i][d] : NAN;
        if (v == v) {
            m = __dmul_rn(m, __dmul_rn(p.mult_w[i], v));
            ++cnt;
        }
    }
    if (cnt == 0) m = 1.0;
    for (int i = 0; i < p.n_add; ++i) {
        const double v = (p.add_col[i] && d < p.attr_cap) ? p.add_col[i][d] : NAN;
        if (v == v) a = __dadd_rn(a, __dmul_rn(p.add_w[i], v));
    }
    p.out64[d] = make_double2(m, a);
    p.out32[d] = make_float2((float)m, (float)a);
    if (m < 0.0) atomicOr(p.negative_flag, 1);
    // non-negative doubles order like their bit patterns
    atomicMax(reinterpret_cast<unsigned long long*>(p.mod_max), (unsigned long long)__double_as_longlong(fabs(m)));
    atomicMax(reinterpret_cast<unsigned long long*>(p.mod_max + 1), (unsigned long long)__double_as_longlong(fabs(a)));
}

__global__ void fill_nan_kernel(double* dst, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = NAN;
}

__global__ void scatter_attr_kernel(double* col, const int32_t* docs, const double* vals, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) col[docs[i]] = vals ? vals[i] : NAN;
}

// (column, document, value) triples in one launch; cols_table[c] = device column pointer
__global__ void scatter_attr_multi_kernel(double* const* cols_table, const int32_t* cols, const int32_t* docs,
                                          const double* vals, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) cols_table[cols[i]][docs[i]] = vals[i];
}

// clear every attribute cell of the listed documents (document overwritten or deleted)
__global__ void clear_attr_kernel(double* const* cols_table, int n_cols, const int32_t* docs, int64_t n, int64_t attr_cap) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t d = docs[i];
    if (d >= attr_cap) return;
    for (int c = 0; c < n_cols; ++c)
        if (cols_table[c]) cols_table[c][d] = NAN;
}

// Merge of all-gathered per-shard lists on the device: one warp per query, candidates strided over the lanes,
// k rounds of warp arg-max under (score desc, doc asc).  Shard s's block: doc int32 [nq,k] | row int32 [nq,k] |
// score f64 [nq,k] packed back to back (the layout b200_index_search_device writes when given one buffer).
__device__ __forceinline__ void warp_merge_shards(const uint8_t* __restrict__ gathered, size_t shard_stride, int nshards,
                                                  int nq, int k, int q, int lane, int32_t* out_doc, int32_t* out_row,
                                                  double* out_score) {
    const int total = nshards * k;
    constexpr int PER = 8;  // up to 256 candidates per query
    double sc[PER];
    int dc[PER], rw[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        const int c = lane + 32 * i;
        sc[i] = -INFINITY;
        dc[i] = INT_MAX;
        rw[i] = -1;
        if (c < total) {
            const int s = c / k, e = c % k;
            const uint8_t* base = gathered + (size_t)s * shard_stride;
            const int d = reinterpret_cast<const int32_t*>(base)[(size_t)q * k + e];
            if (d >= 0) {
                dc[i] = d;
                rw[i] = reinterpret_cast<const int32_t*>(base + (size_t)nq * k * 4)[(size_t)q * k + e];
                sc[i] = reinterpret_cast<const double*>(base + (size_t)nq * k * 8)[(size_t)q * k + e];
            }
        }
    }
    for (int r = 0; r < k; ++r) {
        double bs = -INFINITY;
        int bd = INT_MAX, bi = -1;
#pragma unroll
        for (int i = 0; i < PER; ++i)
            if (sc[i] > bs || (sc[i] == bs && dc[i] < bd)) {
                bs = sc[i];
                bd = dc[i];
                bi = i;
            }
        int br = -1;
#pragma unroll
        for (int i = 0; i < PER; ++i)
            if (i == bi) br = rw[i];
        int owner = lane;
        for (int off = 16; off > 0; off >>= 1) {
            const double os = __shfl_xor_sync(0xffffffffu, bs, off);
            const int od = __shfl_xor_sync(0xffffffffu, bd, off);
            const int orr = __shfl_xor_sync(0xffffffffu, br, off);
            const int oo = __shfl_xor_sync(0xffffffffu, owner, off);
            if (os > bs || (os == bs && od < bd)) {
                bs = os;
                bd = od;
                br = orr;
                owner = oo;
            }
        }
        if (lane == 0) {
            const size_t o = (size_t)q * k + r;
            const bool ok = bd != INT_MAX;
            out_doc[o] = ok ? bd : -1;
            out_row[o] = ok ? br : -1;
            out_score[o] = ok ? bs : -INFINITY;
        }
        if (lane == owner && bi >= 0) {   // retire the winner
#pragma unroll
            for (int i = 0; i < PER; ++i)
                if (i == bi) {
                    sc[i] = -INFINITY;
                    dc[i] = INT_MAX;
                }
        }
    }
}

__global__ void merge_shards_kernel(const uint8_t* __restrict__ gathered, int nshards, int nq, int k, int32_t* out_doc,
                                    int32_t* out_row, double* out_score) {
    const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;
    warp_merge_shards(gathered, (size_t)nq * k * 16, nshards, nq, k, q, lane, out_doc, out_row, out_score);
}

// ------------------------------------------------------------------------------------------------
// Fused exchange + merge over NVLink peer memory (SURVEY §8e: "peer-stores into a symmetric buffer").
// Every rank owns a symmetric exchange buffer [2 parities][world][block] + flags [2][world]; rank r's kernel
//   1. copies its packed local result block into slot r of EVERY peer's buffer (plain stores over NVLink / local),
//   2. publishes it with a system-scope release store of the call's epoch into flag[r] on every peer,
//   3. spins (acquire loads on its OWN flags) until every rank's block of this epoch has landed,
//   4. merges the world * k candidates per query — the same warp_merge_shards as the all-gather path.
// One launch replaces ncclAllGather + merge_shards_kernel; parity = epoch & 1 double-buffers consecutive calls so a
// fast rank's next block never overwrites one a slow rank is still merging.
struct ExchangeParams {
    uint8_t* peer_buf[8];        // peer_buf[s] = base of rank s's exchange buffer mapped into this process
    unsigned long long* peer_flag[8];
    int rank, world;
    int nq, k;
    size_t block_bytes;          // nq * k * 16
    size_t slot_stride;          // bytes between slots (>= block_bytes, 16-byte aligned)
    unsigned long long epoch;
    const uint8_t* local_block;  // packed {doc | row | score} of this rank
    int32_t* out_doc;
    int32_t* out_row;
    double* out_score;
};

__global__ void __launch_bounds__(256) exchange_merge_kernel(ExchangeParams p) {
    const int parity = (int)(p.epoch & 1ull);
    const size_t par_off = (size_t)parity * p.world * p.slot_stride;
    const int n16 = (int)(p.block_bytes / 16);
    const uint4* src = reinterpret_cast<const uint4*>(p.local_block);
    // 1. push: thread t of the grid copies 16-byte words; peers interleaved so every NVLink port sees traffic at once
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
    const int gthreads = gridDim.x * blockDim.x;
    for (int i = gtid; i < n16 * p.world; i += gthreads) {
        const int s = i % p.world, w = i / p.world;
        uint4* dst = reinterpret_cast<uint4*>(p.peer_buf[s] + par_off + (size_t)p.rank * p.slot_stride);
        dst[w] = src[w];
    }
    __threadfence_system();
    __syncthreads();
    // 2. publish: one counter per (peer, source rank); every CTA adds 1, the block is complete at epoch * gridDim.x
    if (threadIdx.x < p.world) {
        unsigned long long* f = p.peer_flag[threadIdx.x] + (size_t)parity * p.world + p.rank;
        asm volatile("red.release.sys.global.add.u64 [%0], %1;" ::"l"(f), "l"(1ull) : "memory");
    }
    // 3. wait for every source rank's block of this epoch
    if (threadIdx.x < p.world) {
        const unsigned long long* f = p.peer_flag[p.rank] + (size_t)parity * p.world + threadIdx.x;
        const unsigned long long want = ((p.epoch >> 1) + 1ull) * (unsigned long long)gridDim.x;
        unsigned long long v;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(f) : "memory");
        } while (v < want);
    }
    __syncthreads();
    // 4. merge: one warp per query
    const uint8_t* mine = p.peer_buf[p.rank] + par_off;
    const int lane = threadIdx.x & 31;
    for (int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); q < p.nq; q += gridDim.x * (blockDim.x >> 5))
        warp_merge_shards(mine, p.slot_stride, p.world, p.nq, p.k, q, lane, p.out_doc, p.out_row, p.out_score);
}

__global__ void fill_empty_kernel(int32_t* out_doc, int32_t* out_row, double* out_score, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        out_doc[i] = -1;
        out_row[i] = -1;
        out_score[i] = -INFINITY;
    }
}

}  // namespace score
}  // namespace mb

// ====================================================================================================
using namespace mb;
using namespace mb::score;

struct b200_exchange {
    int device = 0;
    int rank = 0, world = 1;
    size_t slot_stride = 0;         // bytes per (parity, source rank) slot
    DeviceBuffer<uint8_t> local;    // [2][world][slot_stride] blocks, then [2][world] u64 flags
    IpcMapping mapped[8];           // the other ranks' buffers, opened by b200_exchange_open
    uint8_t* peer[8] = {nullptr};   // peer[s] = rank s's buffer mapped here (peer[rank] == local)
    unsigned long long epoch = 0;
};

struct b200_index {
    int device = 0;
    int dim = 0;
    int metric = 0;
    int sms = 0;
    int64_t capacity = 0;
    int64_t n_rows = 0;
    int64_t dead_rows = 0;  // tombstoned rows still occupying the matrix
    bool has_docs = false;  // false while doc_of_row[i] == i for every row (identity fast path)
    int32_t doc_offset = 0; // added to returned document numbers (shard -> global numbering)
    DeviceBuffer<__half> corpus;       // [capacity, dim]
    DeviceBuffer<int32_t> doc_of_row;  // [capacity]
    DeviceBuffer<float> row_n2;        // [capacity] squared norms (euclidean metric only)
    DeviceBuffer<float> max_n2;        // [1] largest squared norm of a stored row
    DeviceBuffer<int> d_flags;         // [2]: bit 0 of [0] = non-finite / out-of-fp16-range input;
                                       //      [1] = negative multiplier
    // per-search workspaces
    DeviceBuffer<__half> qh;           // [MQ, dim]
    DeviceBuffer<float> q_stage;       // [MQ, dim] fp32 staging for host queries
    DeviceBuffer<float> list_score;    // [grid][MQ][KP]
    DeviceBuffer<int32_t> list_row;
    DeviceBuffer<int32_t> list_doc;
    int out_k = 0;                     // the resident output block holds [MQ, out_k]
    DeviceBuffer<int32_t> o_doc;
    DeviceBuffer<int32_t> o_row;
    DeviceBuffer<double> o_score;
    DeviceBuffer<QState> qs;           // device
    PinnedPtr<QState> h_qs;            // pinned host mirror
    DeviceBuffer<int32_t> cbuf;        // [MQ][ccap] rows appended by the collect pass
    int ccap = 0;
    // score modifiers: per-document numeric attributes (one device column per attribute name, NaN = missing; an empty
    // buffer is a column that was never set)
    std::vector<DeviceBuffer<double>> attr_cols;
    DeviceBuffer<double*> d_cols_table;  // device copy of the attr_cols pointers (B200_MAX_ATTRIBUTE_COLUMNS entries)
    bool cols_table_dirty = true;
    int64_t attr_cap = 0;          // documents each column can hold
    int64_t max_doc = -1;          // largest explicit document number seen by add()
    DeviceBuffer<double2> mod64;   // [mod_cap] (mult, add) of the current modified search
    DeviceBuffer<float2> mod32;
    int64_t mod_cap = 0;
    DeviceBuffer<double> mod_max;  // [2] max |mult|, max |add|
    bool mod_active = false;
    // document filter of the current search (device bitset over local document numbers)
    DeviceBuffer<uint32_t> filter_bits;
    int64_t filter_cap_words = 0;
    int64_t filter_docs = 0;
    uint64_t filter_tag = 0;       // identity of the bitset held in filter_bits (0 = none cached)
    bool filter_active = false;
    // statistics of the exactness machinery (b200_index_search_stats)
    int64_t stat_groups = 0, stat_flagged = 0, stat_collect_passes = 0, stat_host_finalize = 0;
    // scan kernel selection: the streamed-query kernel is forced at any dim (test hook), and the kernel the last scan
    // ran (-1 before the first scan)
    bool force_streamed_q = false;
    int last_scan_kernel = -1;
    // the query group the last scan ran on (debug_last_scan): its size and the scan grid (0 / 0 before any scan)
    int last_nq = 0, last_grid = 0;
    cudaStream_t stream = nullptr;   // own_stream, or the caller's stream set by b200_index_set_stream
    UniqueStream own_stream;
    UniqueEvent ev[4];
    bool timing_valid = false;
    std::mutex mu;
};

namespace {

struct RowArrays {   // the per-row arrays of an index, allocated together for one capacity
    DeviceBuffer<__half> corpus;
    DeviceBuffer<int32_t> doc_of_row;
    DeviceBuffer<float> row_n2;
};

RowArrays alloc_rows(const b200_index* ix, int64_t cap) {
    return {DeviceBuffer<__half>((size_t)cap * ix->dim), DeviceBuffer<int32_t>((size_t)cap),
            ix->metric == B200_METRIC_EUCLIDEAN ? DeviceBuffer<float>((size_t)cap) : DeviceBuffer<float>()};
}

// Replaces the index's row arrays by `r` (capacity `cap`); the caller has copied the rows that stay.
void adopt_rows(b200_index* ix, RowArrays&& r, int64_t cap) {
    ix->corpus = std::move(r.corpus);
    ix->doc_of_row = std::move(r.doc_of_row);
    ix->row_n2 = std::move(r.row_n2);
    ix->capacity = cap;
}

void ensure_capacity(b200_index* ix, int64_t need_rows) {
    if (need_rows <= ix->capacity) return;
    int64_t cap = std::max<int64_t>(need_rows, ix->capacity + ix->capacity / 2);
    cap = (int64_t)round_up((size_t)cap, TILE_N);
    RowArrays r = alloc_rows(ix, cap);
    if (ix->n_rows > 0) {
        MB_CUDA(cudaMemcpyAsync(r.corpus.get(), ix->corpus.get(), (size_t)ix->n_rows * ix->dim * sizeof(__half),
                                cudaMemcpyDeviceToDevice, ix->stream));
        MB_CUDA(cudaMemcpyAsync(r.doc_of_row.get(), ix->doc_of_row.get(), (size_t)ix->n_rows * sizeof(int32_t),
                                cudaMemcpyDeviceToDevice, ix->stream));
        if (r.row_n2)
            MB_CUDA(cudaMemcpyAsync(r.row_n2.get(), ix->row_n2.get(), (size_t)ix->n_rows * sizeof(float),
                                    cudaMemcpyDeviceToDevice, ix->stream));
    }
    MB_CUDA(cudaStreamSynchronize(ix->stream));
    adopt_rows(ix, std::move(r), cap);
}

void ensure_out_k(b200_index* ix, int k) {
    if (k <= ix->out_k) return;
    const int nk = std::max(k, 16);
    MB_CUDA(cudaStreamSynchronize(ix->stream));
    ix->o_doc = DeviceBuffer<int32_t>((size_t)MQ * nk);
    ix->o_row = DeviceBuffer<int32_t>((size_t)MQ * nk);
    ix->o_score = DeviceBuffer<double>((size_t)MQ * nk);
    ix->out_k = nk;
}

void ensure_ccap(b200_index* ix, int cap) {
    if (cap <= ix->ccap) return;
    MB_CUDA(cudaStreamSynchronize(ix->stream));
    ix->cbuf = DeviceBuffer<int32_t>((size_t)MQ * cap);
    ix->ccap = cap;
}

using ScanFn = void (*)(const CUtensorMap, const CUtensorMap, ScanParams);
constexpr int NUM_SCAN_FNS = 16;
// idx bits: 1 docs, 2 bias, 4 modifiers, 8 streamed query block
template <bool C>
ScanFn scan_fn(int idx) {
    static const ScanFn table[NUM_SCAN_FNS] = {
        scan_kernel<false, false, false, C, false>, scan_kernel<true, false, false, C, false>,
        scan_kernel<false, true, false, C, false>,  scan_kernel<true, true, false, C, false>,
        scan_kernel<false, false, true, C, false>,  scan_kernel<true, false, true, C, false>,
        scan_kernel<false, true, true, C, false>,   scan_kernel<true, true, true, C, false>,
        scan_kernel<false, false, false, C, true>,  scan_kernel<true, false, false, C, true>,
        scan_kernel<false, true, false, C, true>,   scan_kernel<true, true, false, C, true>,
        scan_kernel<false, false, true, C, true>,   scan_kernel<true, false, true, C, true>,
        scan_kernel<false, true, true, C, true>,    scan_kernel<true, true, true, C, true>};
    return table[idx];
}

b200_index* index_new(int device, int dim, int metric, int64_t capacity_rows) {
    require_sm90_device(device);
    MB_CHECK_ARG(dim > 0 && dim % BLOCK_K == 0 && dim <= MAX_DIM, "dim must be a multiple of %d and <= %d (got %d)",
                 BLOCK_K, MAX_DIM, dim);
    MB_CHECK_ARG(metric >= 0 && metric <= B200_METRIC_EUCLIDEAN, "unknown metric %d", metric);
    MB_CHECK_ARG(capacity_rows >= 0, "capacity_rows must be >= 0");
    DeviceGuard g(device);
    std::unique_ptr<b200_index> ix(new b200_index());   // released under the guard if the set-up fails
    ix->device = device;
    ix->dim = dim;
    ix->metric = metric;
    ix->sms = std::min(sm_count(device), MAX_LISTS);   // merge_kernel's list-head table holds MAX_LISTS lists
    ix->own_stream = make_stream(cudaStreamNonBlocking);
    ix->stream = ix->own_stream.get();
    for (auto& e : ix->ev) e = make_event();
    ix->qh = DeviceBuffer<__half>((size_t)MQ * dim);
    ix->q_stage = DeviceBuffer<float>((size_t)MQ * dim);
    const size_t nl = (size_t)ix->sms * MQ * KP;
    ix->list_score = DeviceBuffer<float>(nl);
    ix->list_row = DeviceBuffer<int32_t>(nl);
    ix->list_doc = DeviceBuffer<int32_t>(nl);
    ix->qs = DeviceBuffer<QState>(1);
    MB_CUDA(cudaMemset(ix->qs.get(), 0, sizeof(QState)));
    ix->h_qs = make_pinned<QState>();
    ix->max_n2 = DeviceBuffer<float>(1);
    MB_CUDA(cudaMemset(ix->max_n2.get(), 0, sizeof(float)));
    ix->d_flags = DeviceBuffer<int>(2);
    MB_CUDA(cudaMemset(ix->d_flags.get(), 0, 2 * sizeof(int)));
    ix->mod_max = DeviceBuffer<double>(2);
    MB_CUDA(cudaMemset(ix->mod_max.get(), 0, 2 * sizeof(double)));
    ix->d_cols_table = DeviceBuffer<double*>(B200_MAX_ATTRIBUTE_COLUMNS);
    ensure_out_k(ix.get(), 16);
    ensure_ccap(ix.get(), FIN_CAP);
    ensure_capacity(ix.get(), std::max<int64_t>(capacity_rows, TILE_N));
    const auto smem_attr = cudaFuncAttributeMaxDynamicSharedMemorySize;
    for (int i = 0; i < NUM_SCAN_FNS; ++i) {
        MB_CUDA(cudaFuncSetAttribute(scan_fn<false>(i), smem_attr, SMEM_LIMIT));
        MB_CUDA(cudaFuncSetAttribute(scan_fn<true>(i), smem_attr, SMEM_LIMIT));
    }
    MB_CUDA(cudaFuncSetAttribute(merge_kernel, smem_attr, 64 * 1024));
    MB_CUDA(cudaFuncSetAttribute(finalize_kernel, smem_attr, (int)finalize_smem_bytes(FIN_CAP)));
    return ix.release();
}

// Raises B200_ERR_INVALID_ARG when the last conversion saw a non-finite / out-of-fp16-range value (needs a
// synchronised stream).
void check_input_flags(b200_index* ix, const char* what) {
    int flags = 0;
    MB_CUDA(cudaMemcpyAsync(&flags, ix->d_flags.get(), sizeof(int), cudaMemcpyDeviceToHost, ix->stream));
    MB_CUDA(cudaStreamSynchronize(ix->stream));
    if (flags & 1) {
        MB_CUDA(cudaMemsetAsync(ix->d_flags.get(), 0, sizeof(int), ix->stream));
        fail(B200_ERR_INVALID_ARG,
             "%s contain a value that is not finite or does not fit the fp16 row store (|x| <= 65504 after "
             "normalisation)", what);
    }
}

void add_rows_device(b200_index* ix, const float* d_vecs, const int32_t* d_doc_ids, int64_t m) {
    ensure_capacity(ix, ix->n_rows + m);
    const int wpb = 8;
    const int64_t blocks = (m + wpb - 1) / wpb;
    convert_rows_kernel<<<(unsigned)blocks, wpb * 32, 0, ix->stream>>>(
        d_vecs, ix->corpus.get() + (size_t)ix->n_rows * ix->dim, m, ix->dim, m, ix->metric == B200_METRIC_ANGULAR,
        ix->metric == B200_METRIC_EUCLIDEAN ? ix->row_n2.get() + ix->n_rows : nullptr, ix->max_n2.get(),
        ix->d_flags.get());
    MB_CUDA(cudaGetLastError());
    if (d_doc_ids) {
        MB_CUDA(cudaMemcpyAsync(ix->doc_of_row.get() + ix->n_rows, d_doc_ids, (size_t)m * sizeof(int32_t),
                                cudaMemcpyDeviceToDevice, ix->stream));
        ix->has_docs = true;
    } else {
        iota_kernel<<<(unsigned)((m + 255) / 256), 256, 0, ix->stream>>>(ix->doc_of_row.get() + ix->n_rows, m,
                                                                        (int32_t)ix->n_rows);
        MB_CUDA(cudaGetLastError());
    }
    ix->n_rows += m;
}

struct GroupOut {   // device [g, k]
    int32_t* doc;
    int32_t* row;
    double* score;
};

ExactParams exact_params(b200_index* ix, int nq, int k, const GroupOut& out) {
    ExactParams ex{};
    ex.nq = nq;
    ex.k = k;
    ex.dim = ix->dim;
    ex.metric = ix->metric;
    ex.doc_offset = ix->doc_offset;
    ex.qh = ix->qh.get();
    ex.corpus = ix->corpus.get();
    ex.doc_of_row = ix->doc_of_row.get();
    ex.mod64 = ix->mod_active ? ix->mod64.get() : nullptr;
    ex.qs = ix->qs.get();
    ex.out_doc = out.doc;
    ex.out_row = out.row;
    ex.out_score = out.score;
    return ex;
}

struct ScanLaunch {
    CUtensorMap tmap_c, tmap_q;
    ScanParams sp;
    int grid;
    size_t smem;
    int fn_index;
};

ScanLaunch prepare_scan(b200_index* ix, int nq) {
    ScanLaunch L{};
    const int num_tiles = (int)((ix->n_rows + TILE_N - 1) / TILE_N);
    L.grid = std::min(num_tiles, ix->sms);
    const bool mod = ix->mod_active;
    const bool stream_q = ix->dim > RESIDENT_MAX_DIM || ix->force_streamed_q;
    int stages = 16;
    while (stages > 2 && scan_smem_bytes(ix->dim, stages, mod, stream_q) > (size_t)SMEM_LIMIT) --stages;
    L.smem = scan_smem_bytes(ix->dim, stages, mod, stream_q);
    if (L.smem > (size_t)SMEM_LIMIT) fail(B200_ERR_INTERNAL, "scan kernel shared memory budget exceeded");
    L.tmap_c = make_tmap_2d(ix->corpus.get(), CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (uint64_t)ix->dim,
                            (uint64_t)ix->n_rows, (uint64_t)ix->dim * 2, BLOCK_K, TILE_N, CU_TENSOR_MAP_SWIZZLE_128B);
    L.tmap_q = make_tmap_2d(ix->qh.get(), CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (uint64_t)ix->dim, (uint64_t)MQ,
                            (uint64_t)ix->dim * 2, BLOCK_K, MQ, CU_TENSOR_MAP_SWIZZLE_128B);
    ScanParams& sp = L.sp;
    sp.n_rows = (int)ix->n_rows;
    sp.dim = ix->dim;
    sp.num_tiles = num_tiles;
    sp.num_stages = stages;
    sp.nq = nq;
    sp.metric = ix->metric;
    sp.doc_of_row = ix->doc_of_row.get();
    sp.row_bias = ix->row_n2.get();
    sp.mod = mod ? ix->mod32.get() : nullptr;
    sp.filter = ix->filter_active ? ix->filter_bits.get() : nullptr;
    sp.filter_docs = ix->filter_docs;
    sp.qs = ix->qs.get();
    sp.out_score = ix->list_score.get();
    sp.out_row = ix->list_row.get();
    sp.out_doc = ix->list_doc.get();
    sp.cbuf = ix->cbuf.get();
    sp.ccap = ix->ccap;
    const bool bias = ix->metric == B200_METRIC_EUCLIDEAN;
    const bool docs = ix->has_docs || ix->filter_active;   // the filter is applied where the document numbers are read
    L.fn_index = (docs ? 1 : 0) | (bias ? 2 : 0) | (mod ? 4 : 0) | (stream_q ? 8 : 0);
    ix->last_scan_kernel = stream_q ? SCAN_STREAMED_Q : SCAN_RESIDENT_Q;
    ix->last_nq = nq;
    ix->last_grid = L.grid;
    return L;
}

void launch_collect(b200_index* ix, ScanLaunch& L) {
    L.sp.cbuf = ix->cbuf.get();
    L.sp.ccap = ix->ccap;
    scan_fn<true>(L.fn_index)<<<L.grid, THREADS, L.smem, ix->stream>>>(L.tmap_c, L.tmap_q, L.sp);
    MB_CUDA(cudaGetLastError());
}

void launch_finalize(b200_index* ix, int nq, int k, const GroupOut& out) {
    FinalizeParams fp{};
    fp.cbuf = ix->cbuf.get();
    fp.ccap = ix->ccap;
    fp.live_bound = ix->n_rows;
    fp.ex = exact_params(ix, nq, k, out);
    reset_need_kernel<<<1, 1, 0, ix->stream>>>(ix->qs.get());
    finalize_kernel<<<nq, FIN_THREADS, finalize_smem_bytes(std::min(ix->ccap, FIN_CAP)), ix->stream>>>(fp);
    MB_CUDA(cudaGetLastError());
}

void fetch_qstate(b200_index* ix) {
    MB_CUDA(cudaMemcpyAsync(ix->h_qs.get(), ix->qs.get(), sizeof(QState), cudaMemcpyDeviceToHost, ix->stream));
    MB_CUDA(cudaStreamSynchronize(ix->stream));
}

// Exact selection of one query's collected rows on the host (more rows than the device finalize holds in shared
// memory: deep pagination, thousands of exact ties).  Keys are computed on the device (exact_keys_kernel); the
// dedup / sort is the same rule as exact_select, and the query is settled by the device finalize's rule
// (settle_collected).  Returns true when the query needs another collect pass.
bool host_finalize(b200_index* ix, int q, int nq, int k, const GroupOut& out, int cnt) {
    ++ix->stat_host_finalize;
    DeviceBuffer<double> d_dot((size_t)cnt), d_key((size_t)cnt);
    DeviceBuffer<int32_t> d_doc((size_t)cnt);
    GroupOut dummy{nullptr, nullptr, nullptr};
    ExactParams ex = exact_params(ix, nq, k, dummy);
    const int32_t* rows = ix->cbuf.get() + (size_t)q * ix->ccap;
    exact_keys_kernel<<<(cnt + 7) / 8, 256, 0, ix->stream>>>(ex, q, rows, cnt, d_dot.get(), d_key.get(), d_doc.get());
    MB_CUDA(cudaGetLastError());
    struct Hit {
        double dot, key;
        int32_t doc, row;
    };
    std::vector<double> h_dot(cnt), h_key(cnt);
    std::vector<int32_t> h_doc(cnt), h_row(cnt);
    MB_CUDA(cudaMemcpyAsync(h_dot.data(), d_dot.get(), (size_t)cnt * 8, cudaMemcpyDeviceToHost, ix->stream));
    MB_CUDA(cudaMemcpyAsync(h_key.data(), d_key.get(), (size_t)cnt * 8, cudaMemcpyDeviceToHost, ix->stream));
    MB_CUDA(cudaMemcpyAsync(h_doc.data(), d_doc.get(), (size_t)cnt * 4, cudaMemcpyDeviceToHost, ix->stream));
    MB_CUDA(cudaMemcpyAsync(h_row.data(), rows, (size_t)cnt * 4, cudaMemcpyDeviceToHost, ix->stream));
    MB_CUDA(cudaStreamSynchronize(ix->stream));
    std::vector<Hit> v(cnt);
    for (int i = 0; i < cnt; ++i) v[i] = {h_dot[i], h_key[i], h_doc[i], h_row[i]};
    // best chunk per document: (dot desc, row asc); then documents by (key desc, doc asc)
    std::sort(v.begin(), v.end(), [](const Hit& a, const Hit& b) {
        return a.doc < b.doc || (a.doc == b.doc && (a.dot > b.dot || (a.dot == b.dot && a.row < b.row)));
    });
    size_t w = 0;
    for (size_t i = 0; i < v.size(); ++i)
        if (i == 0 || v[i].doc != v[i - 1].doc) v[w++] = v[i];
    v.resize(w);
    std::sort(v.begin(), v.end(), [](const Hit& a, const Hit& b) { return a.key > b.key || (a.key == b.key && a.doc < b.doc); });
    const int nd = (int)v.size();
    QState* h = ix->h_qs.get();
    const double ek = nd >= k ? scan_domain_key(v[k - 1].key, ix->metric, ix->mod_active, h->qn2x[q]) : -INFINITY;
    std::vector<int32_t> o_doc(k, -1), o_row(k, -1);
    std::vector<double> o_sc(k, -std::numeric_limits<double>::infinity());
    for (int i = 0; i < k && i < nd; ++i) {
        o_doc[i] = v[i].doc + ix->doc_offset;
        o_row[i] = v[i].row;
        o_sc[i] = key_score(v[i].key, ix->metric, ix->mod_active);
    }
    MB_CUDA(cudaMemcpyAsync(out.doc + (size_t)q * k, o_doc.data(), (size_t)k * 4, cudaMemcpyHostToDevice, ix->stream));
    MB_CUDA(cudaMemcpyAsync(out.row + (size_t)q * k, o_row.data(), (size_t)k * 4, cudaMemcpyHostToDevice, ix->stream));
    MB_CUDA(cudaMemcpyAsync(out.score + (size_t)q * k, o_sc.data(), (size_t)k * 8, cudaMemcpyHostToDevice, ix->stream));
    MB_CUDA(cudaStreamSynchronize(ix->stream));
    return settle_collected(h, q, k, nd, ek);
}

// One group of <= MQ queries already converted into ix->qh.get().
//   may_sync: the caller tolerates host synchronisation — flagged queries are driven to resolution here.
//   otherwise: one collect + finalize pass is enqueued unconditionally (both exit at once when nothing is flagged);
//   queries still unresolved after it are counted in QState::rounds (b200_index_search_stats).
void search_group(b200_index* ix, int nq, int k, const GroupOut& out, bool record_timing, bool may_sync) {
    const int total = nq * k;
    ++ix->stat_groups;
    if (ix->n_rows == 0) {
        ix->last_nq = ix->last_grid = 0;   // nothing is scanned
        fill_empty_kernel<<<(total + 255) / 256, 256, 0, ix->stream>>>(out.doc, out.row, out.score, total);
        MB_CUDA(cudaGetLastError());
        return;
    }
    query_prep_kernel<<<MQ / 8, 256, 0, ix->stream>>>(ix->qh.get(), ix->dim, ix->metric, ix->mod_active ? 1 : 0,
                                                     ix->max_n2.get(), ix->mod_max.get(), ix->qs.get());
    MB_CUDA(cudaGetLastError());
    ScanLaunch L = prepare_scan(ix, nq);
    if (record_timing) MB_CUDA(cudaEventRecord(ix->ev[0].get(), ix->stream));
    scan_fn<false>(L.fn_index)<<<L.grid, THREADS, L.smem, ix->stream>>>(L.tmap_c, L.tmap_q, L.sp);
    MB_CUDA(cudaGetLastError());
    if (record_timing) MB_CUDA(cudaEventRecord(ix->ev[1].get(), ix->stream));

    MergeParams mp{};
    mp.num_lists = L.grid;
    int sort_n = 32;
    while (sort_n < L.grid * KP) sort_n <<= 1;
    mp.sort_n = sort_n;
    mp.l_only = k > K_MERGE_MAX ? 1 : 0;
    mp.in_score = ix->list_score.get();
    mp.in_row = ix->list_row.get();
    mp.in_doc = ix->list_doc.get();
    mp.ex = exact_params(ix, nq, k, out);
    merge_kernel<<<nq, MERGE_THREADS, (size_t)sort_n * 12, ix->stream>>>(mp);
    MB_CUDA(cudaGetLastError());
    if (record_timing) {
        MB_CUDA(cudaEventRecord(ix->ev[2].get(), ix->stream));
        ix->timing_valid = true;
    }
    if (!may_sync) {
        launch_collect(ix, L);
        launch_finalize(ix, nq, k, out);
        note_unresolved_kernel<<<1, 1, 0, ix->stream>>>(ix->qs.get());
        MB_CUDA(cudaGetLastError());
        return;
    }
    fetch_qstate(ix);
    QState* h = ix->h_qs.get();
    if (h->n_need == 0) return;
    ix->stat_flagged += h->n_need;
    for (int round = 0; h->n_need > 0; ++round) {
        if (round >= 64) fail(B200_ERR_INTERNAL, "exact top-k did not converge in %d collect passes", round);
        ++ix->stat_collect_passes;
        if (round >= 12)   // stop lowering L step by step: take everything
            for (int q = 0; q < nq; ++q)
                if (h->status[q] == Q_NEED) h->L[q] = -INFINITY;
        MB_CUDA(cudaMemcpyAsync(ix->qs.get(), h, sizeof(QState), cudaMemcpyHostToDevice, ix->stream));
        launch_collect(ix, L);
        fetch_qstate(ix);
        int max_cnt = 0;
        for (int q = 0; q < nq; ++q)
            if (h->status[q] == Q_NEED) max_cnt = std::max(max_cnt, h->cnt[q]);
        if (max_cnt > ix->ccap) {   // grow the buffer and repeat the pass with the same thresholds
            if ((size_t)MQ * max_cnt * 4 > ((size_t)8 << 30))
                fail(B200_ERR_OOM, "exact top-k needs %d candidate rows per query (massive ties); not supported", max_cnt);
            ensure_ccap(ix, (int)round_up((size_t)max_cnt + max_cnt / 8, 1024));
            for (int q = 0; q < nq; ++q) h->cnt[q] = 0;
            --round;
            continue;
        }
        if (max_cnt <= FIN_CAP) {
            launch_finalize(ix, nq, k, out);
            fetch_qstate(ix);
        } else {
            int need = 0;
            for (int q = 0; q < nq; ++q)
                if (h->status[q] == Q_NEED && host_finalize(ix, q, nq, k, out, h->cnt[q])) ++need;
            h->n_need = need;
        }
    }
    // leave the device copy clean for the next group (status / thresholds are re-initialised by query_prep_kernel)
}

void convert_queries(b200_index* ix, const float* d_q, int g) {
    convert_rows_kernel<<<MQ / 8, 256, 0, ix->stream>>>(d_q, ix->qh.get(), g, ix->dim, MQ,
                                                        ix->metric == B200_METRIC_ANGULAR, nullptr, nullptr,
                                                        ix->d_flags.get());
    MB_CUDA(cudaGetLastError());
}

void search_device(b200_index* ix, const float* d_q, int nq, int k, int32_t* d_out_doc, int32_t* d_out_row,
                   double* d_out_score, bool may_sync) {
    for (int q0 = 0; q0 < nq; q0 += MQ) {
        const int g = std::min(MQ, nq - q0);
        convert_queries(ix, d_q + (size_t)q0 * ix->dim, g);
        GroupOut out{d_out_doc + (size_t)q0 * k, d_out_row + (size_t)q0 * k, d_out_score + (size_t)q0 * k};
        search_group(ix, g, k, out, q0 + MQ >= nq, may_sync);
    }
}

void check_search_args(const void* q, int nq, int k, const void* a, const void* b, const void* c) {
    MB_CHECK_ARG(q && a && b && c, "NULL buffer");
    MB_CHECK_ARG(nq > 0, "nq must be positive (got %d)", nq);
    MB_CHECK_ARG(k > 0, "k must be positive (got %d)", k);
    MB_CHECK_ARG(k <= 11000, "k = %d exceeds 11000 (Marqo's own limit + offset cap, api/configs.py:24-25)", k);
}

// Largest of the caller's host document ids (-1 when n == 0); a negative id is rejected.
int64_t max_doc_id(const int32_t* doc_ids, int64_t n) {
    int64_t hi = -1;
    for (int64_t i = 0; i < n; ++i) {
        MB_CHECK_ARG(doc_ids[i] >= 0, "doc_ids[%lld] is negative", (long long)i);
        hi = std::max<int64_t>(hi, doc_ids[i]);
    }
    return hi;
}

// largest document number among device-resident ids (ingest path; sizes the score-modifier tables)
void track_max_doc(b200_index* ix, const int32_t* d_ids, int64_t m) {
    std::vector<int32_t> h((size_t)m);
    MB_CUDA(cudaMemcpy(h.data(), d_ids, (size_t)m * sizeof(int32_t), cudaMemcpyDeviceToHost));
    for (int32_t v : h) ix->max_doc = std::max<int64_t>(ix->max_doc, v);
}

int64_t num_docs(const b200_index* ix) { return std::max<int64_t>(ix->n_rows, ix->max_doc + 1); }

void fill_nan(b200_index* ix, double* dst, int64_t n) {
    if (n <= 0) return;
    fill_nan_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ix->stream>>>(dst, n);
    MB_CUDA(cudaGetLastError());
}

void ensure_attr_capacity(b200_index* ix, int64_t need_docs) {
    if (need_docs <= ix->attr_cap) return;
    const int64_t cap = (int64_t)round_up((size_t)std::max<int64_t>(need_docs, ix->attr_cap + ix->attr_cap / 2), 1024);
    for (DeviceBuffer<double>& col : ix->attr_cols) {
        if (!col) continue;
        DeviceBuffer<double> nc((size_t)cap);
        if (ix->attr_cap > 0)
            MB_CUDA(cudaMemcpyAsync(nc.get(), col.get(), (size_t)ix->attr_cap * sizeof(double),
                                    cudaMemcpyDeviceToDevice, ix->stream));
        fill_nan(ix, nc.get() + ix->attr_cap, cap - ix->attr_cap);
        MB_CUDA(cudaStreamSynchronize(ix->stream));
        col = std::move(nc);
    }
    ix->attr_cap = cap;
    ix->cols_table_dirty = true;
}

double* attr_column(b200_index* ix, int column) {
    if ((int)ix->attr_cols.size() <= column) ix->attr_cols.resize(column + 1);
    DeviceBuffer<double>& col = ix->attr_cols[column];
    if (!col) {
        col = DeviceBuffer<double>((size_t)ix->attr_cap);
        fill_nan(ix, col.get(), ix->attr_cap);
        ix->cols_table_dirty = true;
    }
    return col.get();
}

void sync_cols_table(b200_index* ix) {
    if (!ix->cols_table_dirty) return;
    double* table[B200_MAX_ATTRIBUTE_COLUMNS] = {nullptr};
    for (size_t c = 0; c < ix->attr_cols.size(); ++c) table[c] = ix->attr_cols[c].get();
    MB_CUDA(cudaMemcpyAsync(ix->d_cols_table.get(), table, sizeof(table), cudaMemcpyHostToDevice, ix->stream));
    MB_CUDA(cudaStreamSynchronize(ix->stream));   // `table` is a stack array
    ix->cols_table_dirty = false;
}

struct ModScope {  // marks the index as "searching with modifiers" for the duration of one call
    b200_index* ix;
    explicit ModScope(b200_index* i, bool on) : ix(i) { ix->mod_active = on; }
    ~ModScope() { ix->mod_active = false; }
};
struct FilterScope {
    b200_index* ix;
    explicit FilterScope(b200_index* i, bool on) : ix(i) { ix->filter_active = on; }
    ~FilterScope() { ix->filter_active = false; }
};

void prepare_modifiers(b200_index* ix, const int32_t* mult_cols, const double* mult_w, int n_mult,
                       const int32_t* add_cols, const double* add_w, int n_add) {
    const int64_t nd = num_docs(ix);
    if (nd > ix->mod_cap) {
        const int64_t cap = (int64_t)round_up((size_t)nd + (size_t)nd / 2, 1024);
        ix->mod64 = DeviceBuffer<double2>((size_t)cap);
        ix->mod32 = DeviceBuffer<float2>((size_t)cap);
        ix->mod_cap = cap;
    }
    if (nd == 0) return;
    ModifierParams mp{};
    mp.n_docs = (int)nd;
    mp.attr_cap = (int)ix->attr_cap;
    mp.n_mult = n_mult;
    mp.n_add = n_add;
    auto col = [&](int c) -> const double* {
        MB_CHECK_ARG(c >= 0 && c < B200_MAX_ATTRIBUTE_COLUMNS, "attribute column %d out of range", c);
        // a column that was never set is missing everywhere
        return c < (int)ix->attr_cols.size() ? ix->attr_cols[c].get() : nullptr;
    };
    for (int i = 0; i < n_mult; ++i) {
        mp.mult_col[i] = col(mult_cols[i]);
        mp.mult_w[i] = mult_w[i];
    }
    for (int i = 0; i < n_add; ++i) {
        mp.add_col[i] = col(add_cols[i]);
        mp.add_w[i] = add_w[i];
    }
    mp.out64 = ix->mod64.get();
    mp.out32 = ix->mod32.get();
    mp.negative_flag = ix->d_flags.get() + 1;
    mp.mod_max = ix->mod_max.get();
    MB_CUDA(cudaMemsetAsync(ix->d_flags.get() + 1, 0, sizeof(int), ix->stream));
    MB_CUDA(cudaMemsetAsync(ix->mod_max.get(), 0, 2 * sizeof(double), ix->stream));
    modifier_kernel<<<(unsigned)((nd + 255) / 256), 256, 0, ix->stream>>>(mp);
    MB_CUDA(cudaGetLastError());
    int flag = 0;
    MB_CUDA(cudaMemcpyAsync(&flag, ix->d_flags.get() + 1, sizeof(int), cudaMemcpyDeviceToHost, ix->stream));
    MB_CUDA(cudaStreamSynchronize(ix->stream));
    // closeness(field, embeddings) is the best chunk's closeness; the scan keeps, per document, the chunk with the best
    // MODIFIED key, which is the same chunk only while the multiplier is >= 0.
    if (flag && ix->has_docs)
        fail(B200_ERR_UNSUPPORTED,
             "a negative multiplicative score modifier on a corpus with explicit document ids (multi-chunk documents) "
             "is not supported");
}

// Upload the caller's document bitset unless the device already holds the bitset with this tag.
void prepare_filter(b200_index* ix, const uint32_t* bits, int64_t n_docs, uint64_t tag) {
    MB_CHECK_ARG(bits != nullptr && n_docs >= 0, "filter_bits is NULL or filter_docs < 0");
    const int64_t words = (n_docs + 31) / 32;
    if (tag != 0 && tag == ix->filter_tag && n_docs == ix->filter_docs) return;
    if (words > ix->filter_cap_words) {
        MB_CUDA(cudaStreamSynchronize(ix->stream));
        ix->filter_tag = 0;
        const int64_t cap = (int64_t)round_up((size_t)words + (size_t)words / 2 + 1, 256);
        ix->filter_bits = DeviceBuffer<uint32_t>((size_t)cap);
        ix->filter_cap_words = cap;
    }
    if (words > 0)
        MB_CUDA(cudaMemcpyAsync(ix->filter_bits.get(), bits, (size_t)words * 4, cudaMemcpyHostToDevice, ix->stream));
    MB_CUDA(cudaStreamSynchronize(ix->stream));   // the caller's buffer may be pageable and short-lived
    ix->filter_docs = n_docs;
    ix->filter_tag = tag;
}

void search_host(b200_index* ix, const float* q, int nq, int k, int32_t* out_doc, int32_t* out_row, double* out_score) {
    ensure_out_k(ix, k);
    for (int q0 = 0; q0 < nq; q0 += MQ) {
        const int gq = std::min(MQ, nq - q0);
        MB_CUDA(cudaMemcpyAsync(ix->q_stage.get(), q + (size_t)q0 * ix->dim, (size_t)gq * ix->dim * sizeof(float),
                                cudaMemcpyHostToDevice, ix->stream));
        search_device(ix, ix->q_stage.get(), gq, k, ix->o_doc.get(), ix->o_row.get(), ix->o_score.get(), true);
        MB_CUDA(cudaMemcpyAsync(out_doc + (size_t)q0 * k, ix->o_doc.get(), (size_t)gq * k * sizeof(int32_t),
                                cudaMemcpyDeviceToHost, ix->stream));
        MB_CUDA(cudaMemcpyAsync(out_row + (size_t)q0 * k, ix->o_row.get(), (size_t)gq * k * sizeof(int32_t),
                                cudaMemcpyDeviceToHost, ix->stream));
        MB_CUDA(cudaMemcpyAsync(out_score + (size_t)q0 * k, ix->o_score.get(), (size_t)gq * k * sizeof(double),
                                cudaMemcpyDeviceToHost, ix->stream));
        check_input_flags(ix, "queries");   // synchronises
    }
}

void validate_opts(const b200_search_opts* o) {
    if (!o) return;
    MB_CHECK_ARG(o->n_mult >= 0 && o->n_mult <= MAX_MOD_TERMS && o->n_add >= 0 && o->n_add <= MAX_MOD_TERMS,
                 "at most %d multiplicative and %d additive modifiers per search", MAX_MOD_TERMS, MAX_MOD_TERMS);
    MB_CHECK_ARG((o->n_mult == 0 || (o->mult_cols && o->mult_w)) && (o->n_add == 0 || (o->add_cols && o->add_w)),
                 "NULL modifier list");
    for (int i = 0; i < o->n_mult; ++i) MB_CHECK_ARG(std::isfinite(o->mult_w[i]), "mult_w[%d] is not finite", i);
    for (int i = 0; i < o->n_add; ++i) MB_CHECK_ARG(std::isfinite(o->add_w[i]), "add_w[%d] is not finite", i);
    MB_CHECK_ARG(o->filter_bits != nullptr || o->filter_docs == 0, "filter_docs > 0 with filter_bits == NULL");
}

// Body of an index entry point: `body` runs with the index locked and its device current; errors become the
// returned status code.
template <class F>
int with_index(b200_index* ix, const char* null_msg, F&& body) {
    return guarded([&] {
        MB_CHECK_ARG(ix != nullptr, "%s", null_msg);
        std::lock_guard<std::mutex> lk(ix->mu);
        DeviceGuard g(ix->device);
        body();
    });
}
template <class F>
int with_index(b200_index* ix, F&& body) {
    return with_index(ix, "index is NULL", body);
}

// The rows of one add call: vectors and optional document ids (nullptr: row i is document n_rows + i), each in host
// or in device memory.
struct AddRows {
    const float* vecs;
    bool vecs_on_host;
    const int32_t* doc_ids;
    bool ids_on_host;
};

// Body of the add entry points; `args_ok` / `null_msg` is the entry point's own NULL-argument check.  Host vectors
// are staged through the device 64 Ki rows at a time.
int add(b200_index* ix, const AddRows& a, int64_t m, bool args_ok, const char* null_msg) {
    return with_index(ix, [&] {
        MB_CHECK_ARG(m >= 0, "m must be >= 0");
        if (m == 0) return;
        MB_CHECK_ARG(args_ok, "%s", null_msg);
        MB_CHECK_ARG(ix->n_rows + m < (int64_t)INT32_MAX, "row count would exceed 2^31-1");
        const bool host_ids = a.doc_ids && a.ids_on_host;
        const int64_t hi = host_ids ? std::max(ix->max_doc, max_doc_id(a.doc_ids, m)) : ix->max_doc;
        const int64_t chunk = a.vecs_on_host ? std::min<int64_t>(m, 1 << 16) : m;
        DeviceBuffer<float> d_v(a.vecs_on_host ? (size_t)chunk * ix->dim : 0);
        DeviceBuffer<int32_t> d_d(host_ids ? (size_t)chunk : 0);
        const int64_t rows_before = ix->n_rows;   // nothing of a rejected batch stays searchable
        const bool docs_before = ix->has_docs;
        try {
            for (int64_t o = 0; o < m; o += chunk) {
                const int64_t c = std::min(chunk, m - o);
                const float* vecs = a.vecs + (size_t)o * ix->dim;
                const int32_t* ids = a.doc_ids ? a.doc_ids + o : nullptr;
                if (a.vecs_on_host) {
                    MB_CUDA(cudaMemcpyAsync(d_v.get(), vecs, (size_t)c * ix->dim * sizeof(float),
                                            cudaMemcpyHostToDevice, ix->stream));
                    vecs = d_v.get();
                }
                if (host_ids) {
                    MB_CUDA(cudaMemcpyAsync(d_d.get(), ids, (size_t)c * sizeof(int32_t), cudaMemcpyHostToDevice,
                                            ix->stream));
                    ids = d_d.get();
                }
                add_rows_device(ix, vecs, ids, c);
                MB_CUDA(cudaStreamSynchronize(ix->stream));
            }
            check_input_flags(ix, "embeddings");
        } catch (...) {
            ix->n_rows = rows_before;
            ix->has_docs = docs_before;
            throw;
        }
        if (a.doc_ids && !a.ids_on_host) track_max_doc(ix, a.doc_ids, m);
        else ix->max_doc = hi;
    });
}

}  // namespace

void mb::score::debug_scan_kernel(b200_index* ix, int force_streamed, int* last_kernel) {
    MB_CHECK_ARG(ix != nullptr, "index is NULL");
    MB_CHECK_ARG(force_streamed >= -1 && force_streamed <= 1, "force_streamed must be -1, 0 or 1 (got %d)",
                 force_streamed);
    std::lock_guard<std::mutex> lk(ix->mu);
    if (force_streamed >= 0) ix->force_streamed_q = force_streamed != 0;
    if (last_kernel) *last_kernel = ix->last_scan_kernel;
}

// The COLLECT pass and merge_kernel only read the SELECT lists, so after a search they still hold the scan's
// approximate keys; query_prep_kernel is the only writer of eps and nothing writes qh until the next search.
void mb::score::debug_last_scan(b200_index* ix, int* nq, int* grid, float* eps, float* queries, float* list_score,
                                int32_t* list_row, int32_t* list_doc) {
    MB_CHECK_ARG(ix != nullptr, "index is NULL");
    std::lock_guard<std::mutex> lk(ix->mu);
    DeviceGuard g(ix->device);
    MB_CUDA(cudaStreamSynchronize(ix->stream));
    const int n = ix->last_nq, gr = ix->last_grid;
    if (nq) *nq = n;
    if (grid) *grid = gr;
    if (n == 0) return;
    if (eps) {
        std::vector<float> e(MQ);
        MB_CUDA(cudaMemcpy(e.data(), ix->qs.get()->eps, MQ * sizeof(float), cudaMemcpyDeviceToHost));
        std::copy(e.begin(), e.begin() + n, eps);
    }
    if (queries) {
        std::vector<__half> h((size_t)n * ix->dim);
        MB_CUDA(cudaMemcpy(h.data(), ix->qh.get(), h.size() * sizeof(__half), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < h.size(); ++i) queries[i] = __half2float(h[i]);
    }
    // device lists are [grid][MQ][KP]; the caller's are [grid][nq][KP]
    auto lists = [&](void* dst, const void* src, size_t elem) {
        if (!dst) return;
        MB_CUDA(cudaMemcpy2D(dst, (size_t)n * KP * elem, src, (size_t)MQ * KP * elem, (size_t)n * KP * elem, (size_t)gr,
                             cudaMemcpyDeviceToHost));
    };
    lists(list_score, ix->list_score.get(), sizeof(float));
    lists(list_row, ix->list_row.get(), sizeof(int32_t));
    lists(list_doc, ix->list_doc.get(), sizeof(int32_t));
}

extern "C" {

int b200_index_create(int device, int dim, int metric, int64_t capacity_rows, b200_index** out) {
    return guarded([&] {
        MB_CHECK_ARG(out != nullptr, "out is NULL");
        *out = nullptr;
        *out = index_new(device, dim, metric, capacity_rows);
    });
}

int b200_index_destroy(b200_index* ix) {
    return guarded([&] {
        if (!ix) return;
        DeviceGuard g(ix->device);
        delete ix;
    });
}

int b200_index_add(b200_index* ix, const float* vecs, const int32_t* doc_ids, int64_t m) {
    return add(ix, {vecs, true, doc_ids, true}, m, vecs != nullptr, "vecs is NULL");
}

int b200_index_add_device(b200_index* ix, const float* d_vecs, const int32_t* d_doc_ids, int64_t m) {
    return add(ix, {d_vecs, false, d_doc_ids, false}, m, d_vecs != nullptr, "d_vecs is NULL");
}

int b200_index_add_device_docs(b200_index* ix, const float* d_vecs, const int32_t* doc_ids, int64_t m) {
    return add(ix, {d_vecs, false, doc_ids, true}, m, d_vecs != nullptr && doc_ids != nullptr, "NULL argument");
}

int b200_index_delete_doc(b200_index* ix, int32_t doc_id) {
    return with_index(ix, [&] {
        if (ix->n_rows == 0) return;
        tombstone_kernel<<<(unsigned)((ix->n_rows + 255) / 256), 256, 0, ix->stream>>>(ix->doc_of_row.get(), ix->n_rows,
                                                                                      doc_id);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(ix->stream));
        ix->has_docs = true;
    });
}

int b200_index_delete_rows(b200_index* ix, const int32_t* rows, int64_t n) {
    return with_index(ix, [&] {
        MB_CHECK_ARG(n >= 0, "n must be >= 0");
        if (n == 0) return;
        MB_CHECK_ARG(rows != nullptr, "rows is NULL");
        for (int64_t i = 0; i < n; ++i)
            MB_CHECK_ARG(rows[i] >= 0 && rows[i] < ix->n_rows, "rows[%lld] = %d out of range", (long long)i, rows[i]);
        DeviceBuffer<int32_t> d_r((size_t)n);
        MB_CUDA(cudaMemcpyAsync(d_r.get(), rows, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, ix->stream));
        tombstone_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ix->stream>>>(ix->doc_of_row.get(), d_r.get(), n);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(ix->stream));
        ix->has_docs = true;
        ix->dead_rows += n;
    });
}

int b200_index_compact(b200_index* ix, int32_t* out_new_of_old, int64_t* out_rows) {
    return with_index(ix, "NULL argument", [&] {
        MB_CHECK_ARG(out_new_of_old != nullptr && out_rows != nullptr, "NULL argument");
        const int64_t n = ix->n_rows;
        std::vector<int32_t> doc((size_t)n);
        if (n > 0) {
            MB_CUDA(cudaMemcpyAsync(doc.data(), ix->doc_of_row.get(), (size_t)n * 4, cudaMemcpyDeviceToHost,
                                    ix->stream));
            MB_CUDA(cudaStreamSynchronize(ix->stream));
        }
        int64_t live = 0;
        for (int64_t i = 0; i < n; ++i) out_new_of_old[i] = doc[i] >= 0 ? (int32_t)live++ : -1;
        *out_rows = live;
        if (live == n) {
            ix->dead_rows = 0;
            return;
        }
        const int64_t cap = (int64_t)round_up((size_t)std::max<int64_t>(live, TILE_N), TILE_N);
        DeviceBuffer<int32_t> d_map((size_t)n);   // n > live >= 0
        RowArrays r = alloc_rows(ix, cap);
        MB_CUDA(cudaMemcpyAsync(d_map.get(), out_new_of_old, (size_t)n * 4, cudaMemcpyHostToDevice, ix->stream));
        compact_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, ix->stream>>>(
            ix->corpus.get(), r.corpus.get(), ix->doc_of_row.get(), r.doc_of_row.get(), ix->row_n2.get(), r.row_n2.get(),
            d_map.get(), n, ix->dim);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(ix->stream));
        adopt_rows(ix, std::move(r), cap);
        ix->n_rows = live;
        ix->dead_rows = 0;
    });
}

int b200_index_num_rows(b200_index* ix, int64_t* out_rows) {
    return with_index(ix, "NULL argument", [&] {
        MB_CHECK_ARG(out_rows, "NULL argument");
        *out_rows = ix->n_rows;
    });
}

int b200_index_info(b200_index* ix, int* out_dim, int* out_metric, int* out_device) {
    return guarded([&] {
        MB_CHECK_ARG(ix && out_dim && out_metric && out_device, "NULL argument");
        *out_dim = ix->dim;
        *out_metric = ix->metric;
        *out_device = ix->device;
    });
}

int b200_index_get_row(b200_index* ix, int64_t row, float* out_vec) {
    return b200_index_get_rows(ix, &row, 1, out_vec);
}

int b200_index_get_rows(b200_index* ix, const int64_t* rows, int64_t n, float* out_vecs) {
    return with_index(ix, "NULL argument", [&] {
        MB_CHECK_ARG(out_vecs && (rows || n == 0), "NULL argument");
        MB_CHECK_ARG(n >= 0, "n must be >= 0");
        if (n == 0) return;
        std::vector<__half> tmp((size_t)n * ix->dim);
        for (int64_t i = 0; i < n; ++i) {
            MB_CHECK_ARG(rows[i] >= 0 && rows[i] < ix->n_rows, "row %lld out of range", (long long)rows[i]);
            MB_CUDA(cudaMemcpyAsync(tmp.data() + (size_t)i * ix->dim, ix->corpus.get() + (size_t)rows[i] * ix->dim,
                                    (size_t)ix->dim * sizeof(__half), cudaMemcpyDeviceToHost, ix->stream));
        }
        MB_CUDA(cudaStreamSynchronize(ix->stream));
        for (size_t i = 0; i < tmp.size(); ++i) out_vecs[i] = __half2float(tmp[i]);
    });
}

int b200_index_search_ex(b200_index* ix, const float* q, int nq, int k, const b200_search_opts* opts, int32_t* out_doc,
                         int32_t* out_row, double* out_score) {
    return with_index(ix, [&] {
        check_search_args(q, nq, k, out_doc, out_row, out_score);
        validate_opts(opts);
        const bool mod = opts && (opts->n_mult > 0 || opts->n_add > 0);
        const bool filt = opts && opts->filter_bits != nullptr;
        if (mod) prepare_modifiers(ix, opts->mult_cols, opts->mult_w, opts->n_mult, opts->add_cols, opts->add_w, opts->n_add);
        if (filt) prepare_filter(ix, opts->filter_bits, opts->filter_docs, opts->filter_tag);
        ModScope ms(ix, mod);
        FilterScope fs(ix, filt);
        search_host(ix, q, nq, k, out_doc, out_row, out_score);
    });
}

int b200_index_search(b200_index* ix, const float* q, int nq, int k, int32_t* out_doc, int32_t* out_row,
                      double* out_score) {
    return b200_index_search_ex(ix, q, nq, k, nullptr, out_doc, out_row, out_score);
}

int b200_index_search_modified(b200_index* ix, const float* q, int nq, int k, const int32_t* mult_cols,
                               const double* mult_w, int n_mult, const int32_t* add_cols, const double* add_w, int n_add,
                               int32_t* out_doc, int32_t* out_row, double* out_score) {
    b200_search_opts o{};
    o.mult_cols = mult_cols;
    o.mult_w = mult_w;
    o.n_mult = n_mult;
    o.add_cols = add_cols;
    o.add_w = add_w;
    o.n_add = n_add;
    return b200_index_search_ex(ix, q, nq, k, &o, out_doc, out_row, out_score);
}

int b200_index_set_attributes(b200_index* ix, int column, const int32_t* doc_ids, const double* values, int64_t n) {
    return with_index(ix, [&] {
        MB_CHECK_ARG(n >= 0, "n must be >= 0");
        MB_CHECK_ARG(column >= -1 && column < B200_MAX_ATTRIBUTE_COLUMNS, "attribute column %d out of range", column);
        MB_CHECK_ARG(column >= 0 || values == nullptr, "column -1 (all columns) only clears: values must be NULL");
        if (n == 0) return;
        MB_CHECK_ARG(doc_ids != nullptr, "doc_ids is NULL");
        const int64_t hi = max_doc_id(doc_ids, n);
        if (values)
            for (int64_t i = 0; i < n; ++i) MB_CHECK_ARG(std::isfinite(values[i]), "values[%lld] is not finite", (long long)i);
        if (column < 0 && ix->attr_cols.empty()) return;
        ensure_attr_capacity(ix, hi + 1);
        DeviceBuffer<int32_t> d_ids((size_t)n);
        DeviceBuffer<double> d_vals(values ? (size_t)n : 0);
        MB_CUDA(cudaMemcpyAsync(d_ids.get(), doc_ids, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, ix->stream));
        if (values)
            MB_CUDA(cudaMemcpyAsync(d_vals.get(), values, (size_t)n * sizeof(double), cudaMemcpyHostToDevice,
                                    ix->stream));
        const unsigned blocks = (unsigned)((n + 255) / 256);
        if (column >= 0) {
            scatter_attr_kernel<<<blocks, 256, 0, ix->stream>>>(attr_column(ix, column), d_ids.get(), d_vals.get(), n);
            MB_CUDA(cudaGetLastError());
        } else {
            sync_cols_table(ix);
            clear_attr_kernel<<<blocks, 256, 0, ix->stream>>>(ix->d_cols_table.get(), (int)ix->attr_cols.size(),
                                                              d_ids.get(), n, ix->attr_cap);
            MB_CUDA(cudaGetLastError());
        }
        MB_CUDA(cudaStreamSynchronize(ix->stream));
    });
}

int b200_index_set_attributes_multi(b200_index* ix, const int32_t* columns, const int32_t* doc_ids, const double* values,
                                    int64_t n) {
    return with_index(ix, [&] {
        MB_CHECK_ARG(n >= 0, "n must be >= 0");
        if (n == 0) return;
        MB_CHECK_ARG(columns && doc_ids && values, "NULL argument");
        const int64_t hi = max_doc_id(doc_ids, n);
        int max_col = -1;
        for (int64_t i = 0; i < n; ++i) {
            MB_CHECK_ARG(columns[i] >= 0 && columns[i] < B200_MAX_ATTRIBUTE_COLUMNS, "columns[%lld] = %d out of range",
                         (long long)i, columns[i]);
            MB_CHECK_ARG(std::isfinite(values[i]), "values[%lld] is not finite", (long long)i);
            max_col = std::max(max_col, columns[i]);
        }
        ensure_attr_capacity(ix, hi + 1);
        std::vector<char> used(max_col + 1, 0);
        for (int64_t i = 0; i < n; ++i) used[columns[i]] = 1;
        for (int c = 0; c <= max_col; ++c)
            if (used[c]) attr_column(ix, c);
        sync_cols_table(ix);
        DeviceBuffer<int32_t> d_cols((size_t)n), d_ids((size_t)n);
        DeviceBuffer<double> d_vals((size_t)n);
        MB_CUDA(cudaMemcpyAsync(d_cols.get(), columns, (size_t)n * 4, cudaMemcpyHostToDevice, ix->stream));
        MB_CUDA(cudaMemcpyAsync(d_ids.get(), doc_ids, (size_t)n * 4, cudaMemcpyHostToDevice, ix->stream));
        MB_CUDA(cudaMemcpyAsync(d_vals.get(), values, (size_t)n * 8, cudaMemcpyHostToDevice, ix->stream));
        scatter_attr_multi_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ix->stream>>>(
            ix->d_cols_table.get(), d_cols.get(), d_ids.get(), d_vals.get(), n);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(ix->stream));
    });
}

int b200_index_search_device(b200_index* ix, const float* d_q, int nq, int k, int32_t* d_out_doc, int32_t* d_out_row,
                             double* d_out_score, int sync) {
    return with_index(ix, [&] {
        check_search_args(d_q, nq, k, d_out_doc, d_out_row, d_out_score);
        search_device(ix, d_q, nq, k, d_out_doc, d_out_row, d_out_score, sync != 0);
        if (sync) MB_CUDA(cudaStreamSynchronize(ix->stream));
    });
}

int b200_index_search_stats(b200_index* ix, int64_t* out_groups, int64_t* out_flagged, int64_t* out_collect_passes,
                            int64_t* out_unresolved) {
    return with_index(ix, [&] {
        fetch_qstate(ix);
        if (out_groups) *out_groups = ix->stat_groups;
        if (out_flagged) *out_flagged = ix->stat_flagged;
        if (out_collect_passes) *out_collect_passes = ix->stat_collect_passes;
        if (out_unresolved) *out_unresolved = ix->h_qs->rounds;
    });
}

int b200_index_set_stream(b200_index* ix, void* cuda_stream, int use_external) {
    return with_index(ix, [&] {
        MB_CUDA(cudaStreamSynchronize(ix->stream));
        ix->stream = use_external ? reinterpret_cast<cudaStream_t>(cuda_stream) : ix->own_stream.get();
    });
}

int b200_index_set_doc_offset(b200_index* ix, int32_t offset) {
    return with_index(ix, [&] {
        MB_CHECK_ARG(offset >= 0, "offset must be >= 0");
        ix->doc_offset = offset;
    });
}

int b200_topk_merge_device(b200_index* ix, const void* d_gathered, int nshards, int nq, int k, int32_t* d_out_doc,
                           int32_t* d_out_row, double* d_out_score, int sync) {
    return with_index(ix, "NULL argument", [&] {
        MB_CHECK_ARG(d_gathered && d_out_doc && d_out_row && d_out_score, "NULL argument");
        MB_CHECK_ARG(nshards > 0 && nq > 0 && k > 0, "nshards, nq, k must be positive");
        if (nshards * k > 256) fail(B200_ERR_UNSUPPORTED, "device merge handles up to 256 candidates per query");
        merge_shards_kernel<<<(nq + 3) / 4, 128, 0, ix->stream>>>(reinterpret_cast<const uint8_t*>(d_gathered), nshards, nq,
                                                                k, d_out_doc, d_out_row, d_out_score);
        MB_CUDA(cudaGetLastError());
        if (sync) MB_CUDA(cudaStreamSynchronize(ix->stream));
    });
}

int b200_index_last_timing(b200_index* ix, float* scan_ms, float* merge_ms) {
    return with_index(ix, "NULL argument", [&] {
        MB_CHECK_ARG(scan_ms && merge_ms, "NULL argument");
        if (!ix->timing_valid) fail(B200_ERR_INVALID_ARG, "no search has been timed yet");
        MB_CUDA(cudaEventSynchronize(ix->ev[2].get()));
        MB_CUDA(cudaEventElapsedTime(scan_ms, ix->ev[0].get(), ix->ev[1].get()));
        MB_CUDA(cudaEventElapsedTime(merge_ms, ix->ev[1].get(), ix->ev[2].get()));
    });
}

int b200_topk_merge(int nshards, int nq, int k, const int32_t* doc, const int32_t* row, const double* score,
                    int32_t* out_doc, int32_t* out_row, double* out_score) {
    return guarded([&] {
        MB_CHECK_ARG(nshards > 0 && nq > 0 && k > 0, "nshards, nq, k must be positive");
        MB_CHECK_ARG(doc && row && score && out_doc && out_row && out_score, "NULL buffer");
        struct Hit {
            double s;
            int32_t d, r;
        };
        std::vector<Hit> hits;
        for (int q = 0; q < nq; ++q) {
            hits.clear();
            for (int s = 0; s < nshards; ++s)
                for (int i = 0; i < k; ++i) {
                    const size_t o = ((size_t)s * nq + q) * k + i;
                    if (doc[o] >= 0) hits.push_back({score[o], doc[o], row[o]});
                }
            std::sort(hits.begin(), hits.end(),
                      [](const Hit& a, const Hit& b) { return a.s > b.s || (a.s == b.s && a.d < b.d); });
            for (int i = 0; i < k; ++i) {
                const size_t o = (size_t)q * k + i;
                if (i < (int)hits.size()) {
                    out_doc[o] = hits[i].d;
                    out_row[o] = hits[i].r;
                    out_score[o] = hits[i].s;
                } else {
                    out_doc[o] = -1;
                    out_row[o] = -1;
                    out_score[o] = -std::numeric_limits<double>::infinity();
                }
            }
        }
    });
}

// ---------------------------------------------------------------------------------------------------- exchange
int b200_exchange_create(int device, int rank, int world, int max_nq, int max_k, b200_exchange** out, void* out_handle) {
    return guarded([&] {
        MB_CHECK_ARG(out && out_handle, "NULL argument");
        *out = nullptr;
        MB_CHECK_ARG(world >= 1 && world <= 8 && rank >= 0 && rank < world, "bad rank/world %d/%d (world <= 8)", rank, world);
        MB_CHECK_ARG(max_nq > 0 && max_k > 0 && world * max_k <= 256, "world * max_k must be <= 256");
        DeviceGuard g(device);
        std::unique_ptr<b200_exchange> ex(new b200_exchange());
        ex->device = device;
        ex->rank = rank;
        ex->world = world;
        ex->slot_stride = round_up((size_t)max_nq * max_k * 16, 256);
        ex->local =
            DeviceBuffer<uint8_t>(2 * (size_t)world * ex->slot_stride + 2 * (size_t)world * sizeof(unsigned long long));
        MB_CUDA(cudaMemset(ex->local.get(), 0, ex->local.size()));
        MB_CUDA(cudaDeviceSynchronize());
        ex->peer[rank] = ex->local.get();
        cudaIpcMemHandle_t h;
        MB_CUDA(cudaIpcGetMemHandle(&h, ex->local.get()));
        static_assert(sizeof(cudaIpcMemHandle_t) == B200_EXCHANGE_HANDLE_BYTES, "handle size");
        memcpy(out_handle, &h, sizeof(h));
        *out = ex.release();
    });
}

int b200_exchange_open(b200_exchange* ex, const void* handles) {
    return guarded([&] {
        MB_CHECK_ARG(ex && handles, "NULL argument");
        DeviceGuard g(ex->device);
        const uint8_t* hp = reinterpret_cast<const uint8_t*>(handles);
        for (int s = 0; s < ex->world; ++s) {
            if (s == ex->rank || ex->mapped[s]) continue;
            cudaIpcMemHandle_t h;
            memcpy(&h, hp + (size_t)s * B200_EXCHANGE_HANDLE_BYTES, sizeof(h));
            ex->mapped[s] = open_ipc_mapping(h);
            ex->peer[s] = ex->mapped[s].get();
        }
    });
}

int b200_exchange_destroy(b200_exchange* ex) {
    return guarded([&] {
        if (!ex) return;
        DeviceGuard g(ex->device);
        cudaDeviceSynchronize();
        delete ex;
    });
}

int b200_index_search_exchange(b200_index* ix, b200_exchange* ex, const float* d_q, int nq, int k, void* d_local_block,
                               int32_t* d_out_doc, int32_t* d_out_row, double* d_out_score, int sync) {
    return with_index(ix, [&] {
        MB_CHECK_ARG(ex != nullptr && d_local_block != nullptr, "NULL argument");
        check_search_args(d_q, nq, k, d_out_doc, d_out_row, d_out_score);
        MB_CHECK_ARG(nq <= MQ, "one exchange call handles at most %d queries", MQ);
        MB_CHECK_ARG((size_t)nq * k * 16 <= ex->slot_stride, "nq * k exceeds the exchange buffer's block size");
        MB_CHECK_ARG(ex->world * k <= 256, "world * k must be <= 256");
        MB_CHECK_ARG(ex->device == ix->device, "exchange buffer and index live on different devices");
        for (int s = 0; s < ex->world; ++s) MB_CHECK_ARG(ex->peer[s] != nullptr, "peer %d has not been opened", s);
        const size_t nk = (size_t)nq * k;
        uint8_t* blk = reinterpret_cast<uint8_t*>(d_local_block);
        search_device(ix, d_q, nq, k, reinterpret_cast<int32_t*>(blk), reinterpret_cast<int32_t*>(blk + nk * 4),
                      reinterpret_cast<double*>(blk + nk * 8), false);
        ExchangeParams p{};
        for (int s = 0; s < ex->world; ++s) {
            p.peer_buf[s] = ex->peer[s];
            p.peer_flag[s] = reinterpret_cast<unsigned long long*>(ex->peer[s] + 2 * (size_t)ex->world * ex->slot_stride);
        }
        p.rank = ex->rank;
        p.world = ex->world;
        p.nq = nq;
        p.k = k;
        p.block_bytes = nk * 16;
        p.slot_stride = ex->slot_stride;
        p.epoch = ex->epoch++;
        p.local_block = blk;
        p.out_doc = d_out_doc;
        p.out_row = d_out_row;
        p.out_score = d_out_score;
        exchange_merge_kernel<<<8, 256, 0, ix->stream>>>(p);   // the SAME grid on every rank (flag arithmetic)
        MB_CUDA(cudaGetLastError());
        if (sync) MB_CUDA(cudaStreamSynchronize(ix->stream));
    });
}

// ---------------------------------------------------------------------------------------------------- persistence
namespace {
struct FileCloser {
    void operator()(FILE* f) const {
        if (f) fclose(f);
    }
};
struct SnapshotHeader {
    char magic[8];
    int32_t version, dim, metric, has_docs;
    int64_t n_rows;
};
}  // namespace

int b200_index_save(b200_index* ix, const char* path) {
    return with_index(ix, "NULL argument", [&] {
        MB_CHECK_ARG(path, "NULL argument");
        // written under a temporary name and renamed at the end: a crash or a short write never damages the previous
        // snapshot of the same name
        const std::string tmp_path = std::string(path) + ".tmp";
        std::unique_ptr<FILE, FileCloser> f(fopen(tmp_path.c_str(), "wb"));
        if (!f) fail(B200_ERR_INVALID_ARG, "cannot open %s for writing", tmp_path.c_str());
        SnapshotHeader hdr;
        memcpy(hdr.magic, "B200IDX\0", 8);
        hdr.version = 2;   // 2 = version 1 + the attribute-column trailer
        hdr.dim = ix->dim;
        hdr.metric = ix->metric;
        hdr.has_docs = ix->has_docs ? 1 : 0;
        hdr.n_rows = ix->n_rows;
        bool ok = fwrite(&hdr, sizeof(hdr), 1, f.get()) == 1;
        std::vector<uint8_t> buf((size_t)1 << 24);
        auto dump = [&](const void* dptr, size_t bytes) {
            for (size_t o = 0; o < bytes && ok; o += buf.size()) {
                const size_t c = std::min(buf.size(), bytes - o);
                MB_CUDA(cudaMemcpy(buf.data(), (const uint8_t*)dptr + o, c, cudaMemcpyDeviceToHost));
                ok = fwrite(buf.data(), 1, c, f.get()) == c;
            }
        };
        try {
            MB_CUDA(cudaStreamSynchronize(ix->stream));
            dump(ix->corpus.get(), (size_t)ix->n_rows * ix->dim * sizeof(__half));
            dump(ix->doc_of_row.get(), (size_t)ix->n_rows * sizeof(int32_t));
            // trailer: score-modifier attribute columns
            const int64_t trailer[3] = {ix->max_doc, ix->attr_cap, (int64_t)ix->attr_cols.size()};
            ok = ok && fwrite(trailer, sizeof(trailer), 1, f.get()) == 1;
            for (const DeviceBuffer<double>& col : ix->attr_cols) {
                const int32_t present = col ? 1 : 0;
                ok = ok && fwrite(&present, sizeof(present), 1, f.get()) == 1;
                if (col) dump(col.get(), (size_t)ix->attr_cap * sizeof(double));
            }
            ok = ok && fflush(f.get()) == 0;
        } catch (...) {
            f.reset();
            remove(tmp_path.c_str());
            throw;
        }
        FILE* raw = f.release();
        ok = (fclose(raw) == 0) && ok;
        if (!ok) {
            remove(tmp_path.c_str());
            fail(B200_ERR_INTERNAL, "short write to %s", tmp_path.c_str());
        }
        if (rename(tmp_path.c_str(), path) != 0) {
            remove(tmp_path.c_str());
            fail(B200_ERR_INTERNAL, "cannot rename %s to %s", tmp_path.c_str(), path);
        }
    });
}

int b200_index_load(int device, const char* path, b200_index** out) {
    return guarded([&] {
        MB_CHECK_ARG(path && out, "NULL argument");
        *out = nullptr;
        std::unique_ptr<FILE, FileCloser> f(fopen(path, "rb"));
        if (!f) fail(B200_ERR_INVALID_ARG, "cannot open %s", path);
        SnapshotHeader hdr;
        if (fread(&hdr, sizeof(hdr), 1, f.get()) != 1 || memcmp(hdr.magic, "B200IDX\0", 8) != 0 ||
            (hdr.version != 1 && hdr.version != 2))
            fail(B200_ERR_INVALID_ARG, "%s is not a marqo_b200 index snapshot", path);
        require_sm90_device(device);
        DeviceGuard g(device);
        std::unique_ptr<b200_index> owner(index_new(device, hdr.dim, hdr.metric, hdr.n_rows));   // freed under the guard
        b200_index* ix = owner.get();
        std::vector<uint8_t> buf((size_t)1 << 24);
        auto slurp = [&](void* dptr, size_t bytes) {
            for (size_t o = 0; o < bytes; o += buf.size()) {
                const size_t c = std::min(buf.size(), bytes - o);
                if (fread(buf.data(), 1, c, f.get()) != c) fail(B200_ERR_INVALID_ARG, "%s is truncated", path);
                MB_CUDA(cudaMemcpy((uint8_t*)dptr + o, buf.data(), c, cudaMemcpyHostToDevice));
            }
        };
        slurp(ix->corpus.get(), (size_t)hdr.n_rows * hdr.dim * sizeof(__half));
        slurp(ix->doc_of_row.get(), (size_t)hdr.n_rows * sizeof(int32_t));
        ix->n_rows = hdr.n_rows;
        ix->has_docs = hdr.has_docs != 0;
        if (hdr.version >= 2) {
            int64_t trailer[3];
            if (fread(trailer, sizeof(trailer), 1, f.get()) != 1) fail(B200_ERR_INVALID_ARG, "%s is truncated", path);
            MB_CHECK_ARG(trailer[2] >= 0 && trailer[2] <= B200_MAX_ATTRIBUTE_COLUMNS && trailer[1] >= 0,
                         "%s has a corrupt attribute trailer", path);
            ix->max_doc = trailer[0];
            ix->attr_cap = trailer[1];
            ix->attr_cols.resize((size_t)trailer[2]);
            for (DeviceBuffer<double>& col : ix->attr_cols) {
                int32_t present = 0;
                if (fread(&present, sizeof(present), 1, f.get()) != 1) fail(B200_ERR_INVALID_ARG, "%s is truncated", path);
                if (!present) continue;
                col = DeviceBuffer<double>((size_t)ix->attr_cap);
                slurp(col.get(), (size_t)ix->attr_cap * sizeof(double));
            }
            ix->cols_table_dirty = true;
        } else if (ix->has_docs && hdr.n_rows > 0) {
            track_max_doc(ix, ix->doc_of_row.get(), hdr.n_rows);
        }
        if (hdr.n_rows > 0) {   // per-row norms (euclidean) and the largest norm (error bound of the scan)
            row_norms_kernel<<<(unsigned)((hdr.n_rows + 7) / 8), 256, 0, ix->stream>>>(
                ix->corpus.get(), hdr.n_rows, hdr.dim, ix->metric == B200_METRIC_EUCLIDEAN ? ix->row_n2.get() : nullptr,
                ix->max_n2.get());
            MB_CUDA(cudaGetLastError());
            MB_CUDA(cudaStreamSynchronize(ix->stream));
        }
        *out = owner.release();
    });
}

}  // extern "C"
