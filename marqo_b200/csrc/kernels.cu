#include "kernels.cuh"

#include <cmath>
#include <cstdlib>
#include <mutex>
#include <vector>

namespace mb {
namespace kernels {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ------------------------------------------------------------------------------------------------ LayerNorm
// One warp per row, the whole row lives in registers (two-pass mean / variance like torch's CPU kernel).
constexpr int LN_MAX_V4 = 8;        // w <= 1024: every tower but the ViT-H / g / bigG ones
constexpr int LN_WIDE_MAX_V4 = 13;  // w <= 1664: layernorm() only, in its own instantiation so that the rows of up to
                                    // 1024 keep their code (and bits)

template <bool GATHER_EMBED, int MAXV = LN_MAX_V4>
__device__ __forceinline__ void ln_row(float4 (&v)[MAXV], int nv, int w, const float* gamma, const float* beta,
                                       float eps, int lane, float* of, __nv_bfloat16* ob) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
        if (j < nv) s += v[j].x + v[j].y + v[j].z + v[j].w;
    const float mean = warp_sum(s) / (float)w;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
        if (j < nv) {
            const float a = v[j].x - mean, b = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
            q += a * a + b * b + c * c + d * d;
        }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)w + eps);
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
        if (j < nv) {
            const int i4 = lane + 32 * j;
            const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + i4);
            const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + i4);
            float4 y;
            y.x = (v[j].x - mean) * rstd * g.x + b.x;
            y.y = (v[j].y - mean) * rstd * g.y + b.y;
            y.z = (v[j].z - mean) * rstd * g.z + b.z;
            y.w = (v[j].w - mean) * rstd * g.w + b.w;
            if (of) reinterpret_cast<float4*>(of)[i4] = y;
            if (ob) reinterpret_cast<uint2*>(ob)[i4] = make_uint2(pack_bf16x2(y.x, y.y), pack_bf16x2(y.z, y.w));
        }
}

// Elements 4 i4 .. 4 i4 + 3 of a row as fp32: a float4 load, or four bf16 (8 bytes) widened exactly.
__device__ __forceinline__ float4 load4(const float* __restrict__ row, int i4) {
    return reinterpret_cast<const float4*>(row)[i4];
}
__device__ __forceinline__ float4 load4(const __nv_bfloat16* __restrict__ row, int i4) {
    const uint2 u = reinterpret_cast<const uint2*>(row)[i4];
    return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                       __uint_as_float(u.y & 0xffff0000u));
}

// Rows are visited LAST FIRST (block 0 takes the highest rows): the GEMM that produced x wrote its row bands in ascending
// order, so the rows it wrote last — the ones most likely still in the 126 MB L2 — are read first, and the bf16 rows this
// kernel writes last are the low ones the next GEMM (ascending again) starts with.  `reverse` = 0 restores the forward order
// (MARQO_B200_LN_FORWARD=1, A/B timing).  TIn: fp32 rows (the residual stream) or bf16 rows (EVA02's attention output).
template <int MAXV, class TIn = float>
__global__ void __launch_bounds__(256) layernorm_kernel(const TIn* __restrict__ x, long long in_stride,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        float eps, int rows, int w, float* out_f32,
                                                        __nv_bfloat16* out_bf16, int reverse) {
    int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    if (reverse) row = rows - 1 - row;
    const int nv = w / 128;
    const TIn* src = x + (long long)row * in_stride;
    float4 v[MAXV];
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
        if (j < nv) v[j] = load4(src, lane + 32 * j);
    ln_row<false, MAXV>(v, nv, w, gamma, beta, eps, lane, out_f32 ? out_f32 + (long long)row * w : nullptr,
                        out_bf16 ? out_bf16 + (long long)row * w : nullptr);
}

static void check_ln_width(int w, int max_v4 = LN_MAX_V4) {
    if (w % 128 != 0 || w > 128 * max_v4)
        fail(B200_ERR_UNSUPPORTED, "width %d must be a multiple of 128 and <= %d", w, 128 * max_v4);
}

int layernorm(const float* x, long long in_stride, const float* gamma, const float* beta, float eps, int rows, int w,
              float* out_f32, __nv_bfloat16* out_bf16, cudaStream_t s) {
    if (rows <= 0) return 0;
    check_ln_width(w, LN_WIDE_MAX_V4);
    static const int reverse = getenv("MARQO_B200_LN_FORWARD") == nullptr ? 1 : 0;
    if (w <= 128 * LN_MAX_V4)
        layernorm_kernel<LN_MAX_V4>
            <<<(rows + 7) / 8, 256, 0, s>>>(x, in_stride, gamma, beta, eps, rows, w, out_f32, out_bf16, reverse);
    else
        layernorm_kernel<LN_WIDE_MAX_V4>
            <<<(rows + 7) / 8, 256, 0, s>>>(x, in_stride, gamma, beta, eps, rows, w, out_f32, out_bf16, reverse);
    MB_CUDA(cudaGetLastError());
    return 1;
}

int layernorm_bf16(const __nv_bfloat16* x, long long in_stride, const float* gamma, const float* beta, float eps,
                   int rows, int w, __nv_bfloat16* out, cudaStream_t s) {
    if (rows <= 0) return 0;
    check_ln_width(w, LN_WIDE_MAX_V4);
    static const int reverse = getenv("MARQO_B200_LN_FORWARD") == nullptr ? 1 : 0;
    if (w <= 128 * LN_MAX_V4)
        layernorm_kernel<LN_MAX_V4, __nv_bfloat16>
            <<<(rows + 7) / 8, 256, 0, s>>>(x, in_stride, gamma, beta, eps, rows, w, nullptr, out, reverse);
    else
        layernorm_kernel<LN_WIDE_MAX_V4, __nv_bfloat16>
            <<<(rows + 7) / 8, 256, 0, s>>>(x, in_stride, gamma, beta, eps, rows, w, nullptr, out, reverse);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// ------------------------------------------------------------------------------------------------ EVA02, GTE
// Rotary position embedding of q and k in place.  INTERLEAVED (EVA02): one thread rotates 4 pairs (8 bf16 columns) of q
// and the same columns of k of one row; the pair index inside a head is (column % 64) / 2, so 8-column groups never
// straddle a head.  HALF (NewModel's rotate-half): one thread rotates pairs j0 .. j0 + 7 of one head, columns j0 .. j0 + 7
// and j0 + 32 .. j0 + 39, of q and of k.  The first FIRST rows of each sequence (EVA02's class row), and v, are not read
// or written.
template <RopePairing PAIRING, int FIRST>
__global__ void __launch_bounds__(256) rope_qk_kernel(__nv_bfloat16* __restrict__ qkv, int S, int w,
                                                      const float2* __restrict__ table, long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    constexpr bool HALF = PAIRING == RopePairing::HALF;
    const int groups = w / (HALF ? 16 : 8);
    const int g = (int)(i % groups);
    const long long prow = i / groups;                             // rotated row over the batch
    const int pos = (int)(prow % (S - FIRST));                     // its table row
    const long long row = prow + prow / (S - FIRST) * FIRST + FIRST;   // skip each sequence's first FIRST rows
    if constexpr (!HALF) {
        const float4* tab = reinterpret_cast<const float4*>(table + (long long)pos * 32 + (g % 8) * 4);
        const float4 t01 = __ldg(tab), t23 = __ldg(tab + 1);   // (cos, sin) of the 4 pairs
        const float cs[4] = {t01.x, t01.z, t23.x, t23.z}, sn[4] = {t01.y, t01.w, t23.y, t23.w};
#pragma unroll
        for (int part = 0; part < 2; ++part) {   // q, then k
            uint4* p = reinterpret_cast<uint4*>(qkv + row * 3 * w + (long long)part * w) + g;
            const uint4 u = *p;
            uint32_t in[4] = {u.x, u.y, u.z, u.w}, out[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float a = __uint_as_float(in[e] << 16), b = __uint_as_float(in[e] & 0xffff0000u);
                out[e] = pack_bf16x2(a * cs[e] - b * sn[e], b * cs[e] + a * sn[e]);
            }
            *p = make_uint4(out[0], out[1], out[2], out[3]);
        }
    } else {
        const int head = g / 4, j0 = (g % 4) * 8;
        const float4* tab = reinterpret_cast<const float4*>(table + (long long)pos * 32 + j0);
        float cs[8], sn[8];
#pragma unroll
        for (int t = 0; t < 4; ++t) {   // (cos, sin) of pairs j0 + 2t and j0 + 2t + 1
            const float4 v = __ldg(tab + t);
            cs[2 * t] = v.x;
            sn[2 * t] = v.y;
            cs[2 * t + 1] = v.z;
            sn[2 * t + 1] = v.w;
        }
#pragma unroll
        for (int part = 0; part < 2; ++part) {   // q, then k
            __nv_bfloat16* base = qkv + row * 3 * w + (long long)part * w + head * 64 + j0;
            uint4* pa = reinterpret_cast<uint4*>(base);        // the first halves a of the 8 pairs
            uint4* pb = reinterpret_cast<uint4*>(base + 32);   // their second halves b
            const uint4 ua = *pa, ub = *pb;
            const uint32_t ia[4] = {ua.x, ua.y, ua.z, ua.w}, ib[4] = {ub.x, ub.y, ub.z, ub.w};
            uint32_t oa[4], ob[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float a0 = __uint_as_float(ia[e] << 16), a1 = __uint_as_float(ia[e] & 0xffff0000u);
                const float b0 = __uint_as_float(ib[e] << 16), b1 = __uint_as_float(ib[e] & 0xffff0000u);
                const float c0 = cs[2 * e], s0 = sn[2 * e], c1 = cs[2 * e + 1], s1 = sn[2 * e + 1];
                oa[e] = pack_bf16x2(a0 * c0 - b0 * s0, a1 * c1 - b1 * s1);
                ob[e] = pack_bf16x2(b0 * c0 + a0 * s0, b1 * c1 + a1 * s1);
            }
            *pa = make_uint4(oa[0], oa[1], oa[2], oa[3]);
            *pb = make_uint4(ob[0], ob[1], ob[2], ob[3]);
        }
    }
}

void rope_table(int G, int ref, float* out) {
    const double s = (double)ref / G;
    for (int r = 0; r < G; ++r)
        for (int c = 0; c < G; ++c)
            for (int i = 0; i < 32; ++i) {
                const double theta = (i < 16 ? r : c) * s * std::pow(10000.0, -(double)(i % 16) / 16.0);
                float* o = out + ((long long)(r * G + c) * 32 + i) * 2;
                o[0] = (float)std::cos(theta);
                o[1] = (float)std::sin(theta);
            }
}

void rope_table_ntk(int ctx, double base, double factor, float* out) {
    for (int j = 0; j < 32; ++j) {
        const double f = std::pow(base * factor, -2.0 * j / 64.0) / std::pow(factor, 2.0 / 64.0);
        for (int s = 0; s < ctx; ++s) {
            float* o = out + ((long long)s * 32 + j) * 2;
            o[0] = (float)std::cos(s * f);
            o[1] = (float)std::sin(s * f);
        }
    }
}

template <RopePairing PAIRING, int FIRST>
void launch_rope_qk(__nv_bfloat16* qkv, int S, int w, const float* table, long long total, cudaStream_t s) {
    rope_qk_kernel<PAIRING, FIRST><<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
        qkv, S, w, reinterpret_cast<const float2*>(table), total);
}

int rope_qk(__nv_bfloat16* qkv, int n, int S, int first, int w, const float* table, RopePairing pairing,
            cudaStream_t s) {
    if (first != 0 && first != 1) fail(B200_ERR_INTERNAL, "rope_qk: first rotated row %d must be 0 or 1", first);
    if (n <= 0 || S <= first) return 0;
    if (w % 64 != 0) fail(B200_ERR_UNSUPPORTED, "rope_qk: width %d must be a multiple of 64", w);
    const bool half = pairing == RopePairing::HALF;
    const long long total = (long long)n * (S - first) * (w / (half ? 16 : 8));
    if (half)
        first ? launch_rope_qk<RopePairing::HALF, 1>(qkv, S, w, table, total, s)
              : launch_rope_qk<RopePairing::HALF, 0>(qkv, S, w, table, total, s);
    else
        first ? launch_rope_qk<RopePairing::INTERLEAVED, 1>(qkv, S, w, table, total, s)
              : launch_rope_qk<RopePairing::INTERLEAVED, 0>(qkv, S, w, table, total, s);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// GeGLU: one thread per 8 columns of a row, reading the up and gate groups before writing over the up group, so out may
// be the up half of in itself (ldo = 2h).
__global__ void __launch_bounds__(256) geglu_kernel(const __nv_bfloat16* in, int h, __nv_bfloat16* out, long long ldo,
                                                    long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int groups = h / 8;
    const long long row = i / groups;
    const int c8 = (int)(i % groups);
    const uint4 uv = reinterpret_cast<const uint4*>(in + row * 2 * h)[c8];
    const uint4 gv = reinterpret_cast<const uint4*>(in + row * 2 * h + h)[c8];
    const uint32_t uw[4] = {uv.x, uv.y, uv.z, uv.w}, gw[4] = {gv.x, gv.y, gv.z, gv.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float y[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float u = __uint_as_float(k ? uw[e] & 0xffff0000u : uw[e] << 16);
            const float g = __uint_as_float(k ? gw[e] & 0xffff0000u : gw[e] << 16);
            // torch's exact GELU: g / 2 (1 + erf(g / sqrt 2))
            y[k] = 0.5f * g * (1.0f + erff(g * 0.70710678118654752440f)) * u;
        }
        o[e] = pack_bf16x2(y[0], y[1]);
    }
    reinterpret_cast<uint4*>(out + row * ldo)[c8] = make_uint4(o[0], o[1], o[2], o[3]);
}

int geglu(const __nv_bfloat16* in, int rows, int h, __nv_bfloat16* out, long long ldo, cudaStream_t s) {
    if (rows <= 0) return 0;
    if (h <= 0 || h % 8 != 0) fail(B200_ERR_UNSUPPORTED, "geglu: hidden size %d must be a positive multiple of 8", h);
    if (ldo < h || ldo % 8 != 0) fail(B200_ERR_INTERNAL, "geglu: ldo %lld", ldo);
    const long long total = (long long)rows * (h / 8);
    geglu_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, h, out, ldo, total);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// SwiGLU + LayerNorm: one 128-thread block per row, each thread holding up to SWIGLU_V groups of 8 hidden columns in
// registers.  The whole row is read before any of it is written, so out may be the gate half of in (ldo = 2 hp).
constexpr int SWIGLU_THREADS = 128, SWIGLU_V = 3;
static_assert(SWIGLU_THREADS * SWIGLU_V * 8 == SWIGLU_MAX_HP, "swiglu_ln's registers hold SWIGLU_MAX_HP columns");

__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();   // red may still be read from the previous sum
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < SWIGLU_THREADS / 32; ++i) t += red[i];
    return t;
}

__global__ void __launch_bounds__(SWIGLU_THREADS) swiglu_ln_kernel(const __nv_bfloat16* in, int hp, int h,
                                                                    const float* __restrict__ gamma,
                                                                    const float* __restrict__ beta, float eps,
                                                                    __nv_bfloat16* out, long long ldo) {
    __shared__ float red[SWIGLU_THREADS / 32];
    const long long row = blockIdx.x;
    const __nv_bfloat16* g_row = in + row * 2 * hp;
    const __nv_bfloat16* x_row = g_row + hp;
    const int groups = hp / 8;
    float u[SWIGLU_V][8];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < SWIGLU_V; ++j) {
        const int c8 = threadIdx.x + SWIGLU_THREADS * j;
        if (c8 < groups) {
            const uint4 gv = reinterpret_cast<const uint4*>(g_row)[c8];
            const uint4 xv = reinterpret_cast<const uint4*>(x_row)[c8];
            const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w}, xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const uint32_t gb = gw[e / 2], xb = xw[e / 2];
                const float gf = __uint_as_float(e % 2 ? gb & 0xffff0000u : gb << 16);
                const float xf = __uint_as_float(e % 2 ? xb & 0xffff0000u : xb << 16);
                // SiLU(g) x = g x / (1 + e^-g); the pad columns (zero weights and bias) give exactly 0
                u[j][e] = gf / (1.0f + expf(-gf)) * xf;
                if (c8 * 8 + e < h) s += u[j][e];
            }
        }
    }
    const float mean = block_sum(s, red) / (float)h;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < SWIGLU_V; ++j) {
        const int c8 = threadIdx.x + SWIGLU_THREADS * j;
        if (c8 < groups)
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (c8 * 8 + e < h) {
                    const float d = u[j][e] - mean;
                    q += d * d;
                }
    }
    const float rstd = 1.0f / sqrtf(block_sum(q, red) / (float)h + eps);
    __nv_bfloat16* o_row = out + row * ldo;
#pragma unroll
    for (int j = 0; j < SWIGLU_V; ++j) {
        const int c8 = threadIdx.x + SWIGLU_THREADS * j;
        if (c8 < groups) {
            float y[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int c = c8 * 8 + e;
                y[e] = c < h ? (u[j][e] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c) : 0.f;
            }
            reinterpret_cast<uint4*>(o_row)[c8] = make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]),
                                                             pack_bf16x2(y[4], y[5]), pack_bf16x2(y[6], y[7]));
        }
    }
}

int swiglu_ln(const __nv_bfloat16* in, int rows, int hp, int h, const float* gamma, const float* beta, float eps,
              __nv_bfloat16* out, long long ldo, cudaStream_t s) {
    if (rows <= 0) return 0;
    if (hp % 64 != 0 || hp > SWIGLU_MAX_HP || h <= hp - 64 || h > hp)
        fail(B200_ERR_UNSUPPORTED, "swiglu_ln: hidden %d padded to %d must round up to a multiple of 64, <= %d", h, hp,
             SWIGLU_MAX_HP);
    if (ldo < hp || ldo % 8 != 0) fail(B200_ERR_INTERNAL, "swiglu_ln: ldo %lld", ldo);
    swiglu_ln_kernel<<<(unsigned)rows, SWIGLU_THREADS, 0, s>>>(in, hp, h, gamma, beta, eps, out, ldo);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// ------------------------------------------------------------------------------------------------ im2col
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ chw, int n, int S, int p, int kpad,
                                                     int cls, __nv_bfloat16* __restrict__ out) {
    // one thread = 8 consecutive k of one token row; the class-token row (t < cls) of each image is zero
    const int g = S / p;
    const int tokens = g * g + cls;
    const int groups = kpad / 8;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)n * tokens * groups;
    if (gid >= total) return;
    const int kg = (int)(gid % groups);
    const long long row = gid / groups;
    const long long b = row / tokens;
    const int t = (int)(row - b * tokens) - cls;
    const int px = t % g, py = t / g;
    const int K = 3 * p * p;
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int k = kg * 8 + e;
        float val = 0.f;
        if (t >= 0 && k < K) {
            const int c = k / (p * p);
            const int rem = k - c * p * p;
            const int dy = rem / p, dx = rem - dy * p;
            const int y = py * p + dy, x = px * p + dx;
            val = chw[((b * 3 + c) * S + y) * S + x];
        }
        f[e] = val;
    }
    reinterpret_cast<uint4*>(out)[gid] =
        make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

int im2col_f32(const float* chw, int n, int S, int p, int kpad, int cls, __nv_bfloat16* out, cudaStream_t s) {
    if (n <= 0) return 0;
    const int g = S / p;
    const long long total = (long long)n * (g * g + cls) * (kpad / 8);
    im2col_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(chw, n, S, p, kpad, cls, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// ------------------------------------------------------------------------------------------------ embeddings
__global__ void __launch_bounds__(256) vit_embed_kernel(float4* __restrict__ x, const float4* __restrict__ cls,
                                                        const float4* __restrict__ pos, long long total,
                                                        int tokens_per_image, int w4) {
    // one thread = 4 columns of one token row
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const long long row = i / w4;
    const int c = (int)(i - row * w4), t = (int)(row % tokens_per_image);
    float4 v = __ldg(pos + (long long)t * w4 + c);
    if (t == 0 && cls != nullptr) {
        const float4 a = __ldg(cls + c);
        v = make_float4(a.x + v.x, a.y + v.y, a.z + v.z, a.w + v.w);
    }
    x[i] = v;
}

int vit_embed_rows(float* x, const float* cls, const float* pos, int n, int tokens_per_image, int w, cudaStream_t s) {
    if (n <= 0) return 0;
    const long long total = (long long)n * tokens_per_image * (w / 4);
    vit_embed_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
        reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(cls), reinterpret_cast<const float4*>(pos), total,
        tokens_per_image, w / 4);
    MB_CUDA(cudaGetLastError());
    return 1;
}

__global__ void __launch_bounds__(256) clip_text_embed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ tok,
                                                              const float* __restrict__ pos, int n, int S, int w, int vocab,
                                                              float* __restrict__ x, int32_t* __restrict__ eot) {
    // one warp per token row
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= (long long)n * S) return;
    const int s = (int)(row % S);
    int id = ids[row];
    id = min(max(id, 0), vocab - 1);
    const float4* t4 = reinterpret_cast<const float4*>(tok + (long long)id * w);
    const float4* p4 = reinterpret_cast<const float4*>(pos + (long long)s * w);
    float4* o4 = reinterpret_cast<float4*>(x + row * w);
    for (int i = lane; i < w / 4; i += 32) {
        const float4 a = __ldg(t4 + i), b = __ldg(p4 + i);
        o4[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    if (s == 0 && lane == 0) {
        // torch.argmax: first occurrence of the maximum id
        const int32_t* r = ids + row;
        int best = 0, bv = r[0];
        for (int j = 1; j < S; ++j)
            if (r[j] > bv) {
                bv = r[j];
                best = j;
            }
        eot[row / S] = best;
    }
}

int clip_text_embed(const int32_t* ids, const float* tok, const float* pos, int n, int S, int w, int vocab, float* x,
                    int32_t* eot, cudaStream_t s) {
    if (n <= 0) return 0;
    const long long rows = (long long)n * S;
    clip_text_embed_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(ids, tok, pos, n, S, w, vocab, x, eot);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// POS: BERT's position_embeddings row s is added; GTE (NewModel, rotary positions) has no position table.
template <bool POS>
__global__ void __launch_bounds__(256) bert_embed_ln_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ mask,
                                                            const float* __restrict__ word, const float* __restrict__ pos,
                                                            const float* __restrict__ type0, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float eps, int n, int S, int w,
                                                            int vocab, float* __restrict__ x, __nv_bfloat16* __restrict__ h,
                                                            int32_t* __restrict__ kv_len) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= (long long)n * S) return;
    const int s = (int)(row % S);
    int id = ids[row];
    id = min(max(id, 0), vocab - 1);
    const int nv = w / 128;
    const float4* w4 = reinterpret_cast<const float4*>(word + (long long)id * w);
    const float4* t4 = reinterpret_cast<const float4*>(type0);
    float4 v[LN_MAX_V4];
    if constexpr (POS) {
        const float4* p4 = reinterpret_cast<const float4*>(pos + (long long)s * w);
#pragma unroll
        for (int j = 0; j < LN_MAX_V4; ++j)
            if (j < nv) {
                const int i4 = lane + 32 * j;
                const float4 a = __ldg(w4 + i4), b = __ldg(p4 + i4), c = __ldg(t4 + i4);
                // HF: inputs_embeds + token_type_embeddings, then + position_embeddings
                v[j] = make_float4((a.x + c.x) + b.x, (a.y + c.y) + b.y, (a.z + c.z) + b.z, (a.w + c.w) + b.w);
            }
    } else {
#pragma unroll
        for (int j = 0; j < LN_MAX_V4; ++j)
            if (j < nv) {
                const int i4 = lane + 32 * j;
                const float4 a = __ldg(w4 + i4), c = __ldg(t4 + i4);
                v[j] = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);   // NewEmbeddings: word + token type
            }
    }
    ln_row<true>(v, nv, w, gamma, beta, eps, lane, x + row * w, h + row * w);
    if (s == 0 && lane == 0) {
        int cnt = S;
        if (mask) {
            cnt = 0;
            for (int j = 0; j < S; ++j) cnt += mask[row + j] != 0;
        }
        kv_len[row / S] = cnt;
    }
}

int bert_embed_ln(const int32_t* ids, const int32_t* mask, const float* word, const float* pos, const float* type0,
                  const float* gamma, const float* beta, float eps, int n, int S, int w, int vocab, float* x,
                  __nv_bfloat16* h, int32_t* kv_len, cudaStream_t s) {
    if (n <= 0) return 0;
    check_ln_width(w);
    const long long rows = (long long)n * S;
    const unsigned blocks = (unsigned)((rows + 7) / 8);
    if (pos)
        bert_embed_ln_kernel<true><<<blocks, 256, 0, s>>>(ids, mask, word, pos, type0, gamma, beta, eps, n, S, w, vocab, x,
                                                           h, kv_len);
    else
        bert_embed_ln_kernel<false><<<blocks, 256, 0, s>>>(ids, mask, word, nullptr, type0, gamma, beta, eps, n, S, w,
                                                            vocab, x, h, kv_len);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// TYPE_ROW: XLM-R adds token_type_embeddings row 0 (HF: (inputs_embeds + token_type) + position, as BERT); MPNet has none.
template <bool TYPE_ROW>
__global__ void __launch_bounds__(256) roberta_embed_ln_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ mask,
                                                               const float* __restrict__ word, const float* __restrict__ pos,
                                                               const float* __restrict__ type0, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, float eps, int n, int S, int w,
                                                               int vocab, int pad, float* __restrict__ x,
                                                               __nv_bfloat16* __restrict__ h, int32_t* __restrict__ kv_len) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= (long long)n * S) return;
    const int s = (int)(row % S);
    const int32_t* seq = ids + (row - s);
    // HF create_position_ids_from_input_ids: cumsum(ids != pad) * (ids != pad) + pad, from the ids, not the mask
    int cnt = 0;
    for (int j = lane; j <= s; j += 32) cnt += seq[j] != pad;
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    int id = ids[row];
    const int p = id != pad ? pad + cnt : pad;
    id = min(max(id, 0), vocab - 1);
    const int nv = w / 128;
    const float4* w4 = reinterpret_cast<const float4*>(word + (long long)id * w);
    const float4* p4 = reinterpret_cast<const float4*>(pos + (long long)p * w);
    const float4* t4 = reinterpret_cast<const float4*>(type0);
    float4 v[LN_MAX_V4];
#pragma unroll
    for (int j = 0; j < LN_MAX_V4; ++j)
        if (j < nv) {
            const int i4 = lane + 32 * j;
            float4 a = __ldg(w4 + i4);
            const float4 b = __ldg(p4 + i4);
            if (TYPE_ROW) {
                const float4 c = __ldg(t4 + i4);
                a = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);
            }
            v[j] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);   // HF: inputs_embeds (+ type) + position
        }
    ln_row<true>(v, nv, w, gamma, beta, eps, lane, x + row * w, h + row * w);
    if (s == 0 && lane == 0) {
        int c = S;
        if (mask) {
            c = 0;
            for (int j = 0; j < S; ++j) c += mask[row + j] != 0;
        }
        kv_len[row / S] = c;
    }
}

int roberta_embed_ln(const int32_t* ids, const int32_t* mask, const float* word, const float* pos, const float* type0,
                     const float* gamma, const float* beta, float eps, int n, int S, int w, int vocab, int pad, float* x,
                     __nv_bfloat16* h, int32_t* kv_len, cudaStream_t s) {
    if (n <= 0) return 0;
    check_ln_width(w);
    const long long rows = (long long)n * S;
    const unsigned blocks = (unsigned)((rows + 7) / 8);
    if (type0)
        roberta_embed_ln_kernel<true><<<blocks, 256, 0, s>>>(ids, mask, word, pos, type0, gamma, beta, eps, n, S, w, vocab,
                                                             pad, x, h, kv_len);
    else
        roberta_embed_ln_kernel<false><<<blocks, 256, 0, s>>>(ids, mask, word, pos, nullptr, gamma, beta, eps, n, S, w,
                                                              vocab, pad, x, h, kv_len);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// ------------------------------------------------------------------------------------------------ heads
__device__ __forceinline__ float block_sum_256(float v, float* red) {
    v = warp_sum(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i];
    return t;
}

// CLIP head in three small kernels with enough parallelism to be latency-free:
//   (1) head_ln_kernel      one warp per image: gather the pooled token row, LayerNorm -> pooled fp32 [n, w]
//   (2) head_proj_kernel    grid (n/4, E/64): 4 images x 64 outputs per CTA, K split over 4 thread groups
//   (3) head_norm_kernel    one warp per image: L2 normalise (no epsilon, abstract_clip_model.py:83-85)
constexpr int HEAD_IMGS = 4;
constexpr int HEAD_COLS = 64;

__global__ void __launch_bounds__(256) head_ln_kernel(const float* __restrict__ x, int S, const int32_t* __restrict__ row_in_seq,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      float eps, int n, int w, float* __restrict__ pooled) {
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= n) return;
    const int r = row_in_seq ? row_in_seq[b] : 0;
    const float* src = x + ((long long)b * S + r) * w;
    float s = 0.f;
    for (int i = lane; i < w; i += 32) s += src[i];
    const float mean = warp_sum(s) / (float)w;
    float q = 0.f;
    for (int i = lane; i < w; i += 32) {
        const float d = src[i] - mean;
        q += d * d;
    }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)w + eps);
    for (int i = lane; i < w; i += 32) pooled[(long long)b * w + i] = (src[i] - mean) * rstd * gamma[i] + beta[i];
}

__global__ void __launch_bounds__(256) head_proj_kernel(const float* __restrict__ pooled, const float* __restrict__ proj, int n,
                                                        int w, int E, float* __restrict__ out) {
    __shared__ float part[4][HEAD_IMGS][HEAD_COLS];
    extern __shared__ float s_pool[];   // [HEAD_IMGS][w]
    const int b0 = blockIdx.x * HEAD_IMGS;
    const int e = blockIdx.y * HEAD_COLS + (threadIdx.x & (HEAD_COLS - 1));
    const int slice = threadIdx.x >> 6;   // 4 K-slices
    for (int i = threadIdx.x; i < HEAD_IMGS * w; i += 256) {
        const int k = i / w, c = i - k * w;
        s_pool[i] = b0 + k < n ? pooled[(long long)(b0 + k) * w + c] : 0.f;
    }
    __syncthreads();
    float acc[HEAD_IMGS];
#pragma unroll
    for (int k = 0; k < HEAD_IMGS; ++k) acc[k] = 0.f;
    const int i0 = slice * (w / 4), i1 = i0 + w / 4;
    if (e < E) {
#pragma unroll 8
        for (int i = i0; i < i1; ++i) {
            const float pj = __ldg(proj + (long long)i * E + e);
#pragma unroll
            for (int k = 0; k < HEAD_IMGS; ++k) acc[k] = fmaf(s_pool[k * w + i], pj, acc[k]);
        }
    }
#pragma unroll
    for (int k = 0; k < HEAD_IMGS; ++k) part[slice][k][threadIdx.x & (HEAD_COLS - 1)] = acc[k];
    __syncthreads();
    if (slice == 0 && e < E) {
#pragma unroll
        for (int k = 0; k < HEAD_IMGS; ++k)
            if (b0 + k < n) {
                const int c = threadIdx.x & (HEAD_COLS - 1);
                // fixed order: the result does not depend on scheduling
                out[(long long)(b0 + k) * E + e] = ((part[0][k][c] + part[1][k][c]) + part[2][k][c]) + part[3][k][c];
            }
    }
}

__global__ void __launch_bounds__(256) head_norm_kernel(float* __restrict__ out, int n, int E) {
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= n) return;
    float* row = out + (long long)b * E;
    float ss = 0.f;
    for (int i = lane; i < E; i += 32) ss += row[i] * row[i];
    const float nrm = sqrtf(warp_sum(ss));
    for (int i = lane; i < E; i += 32) row[i] = row[i] / nrm;
}

int clip_head(const float* x, int S, const int32_t* row_in_seq, const float* gamma, const float* beta, float eps,
              const float* proj, int n, int w, int E, int normalize, float* out, float* pooled_ws, cudaStream_t s) {
    if (n <= 0) return 0;
    if (w % 4 != 0 || (size_t)HEAD_IMGS * w * sizeof(float) > 40 * 1024)
        fail(B200_ERR_UNSUPPORTED, "clip_head: width %d unsupported", w);
    head_ln_kernel<<<(n + 7) / 8, 256, 0, s>>>(x, S, row_in_seq, gamma, beta, eps, n, w, pooled_ws);
    MB_CUDA(cudaGetLastError());
    const dim3 grid((n + HEAD_IMGS - 1) / HEAD_IMGS, (E + HEAD_COLS - 1) / HEAD_COLS);
    head_proj_kernel<<<grid, 256, (size_t)HEAD_IMGS * w * sizeof(float), s>>>(pooled_ws, proj, n, w, E, out);
    MB_CUDA(cudaGetLastError());
    if (!normalize) return 2;
    head_norm_kernel<<<(n + 7) / 8, 256, 0, s>>>(out, n, E);
    MB_CUDA(cudaGetLastError());
    return 3;
}

__global__ void __launch_bounds__(256) bert_head_kernel(const float* __restrict__ x, const int32_t* __restrict__ kv_len, int S,
                                                        int w, int pool, int normalize, float* __restrict__ out) {
    __shared__ float red[8];
    const int b = blockIdx.x;
    const int len = min(max(kv_len[b], 0), S);
    const float* src = x + (long long)b * S * w;
    float vals[4];  // w <= 1024
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int i = threadIdx.x + 256 * j;
        float v = 0.f;
        if (i < w) {
            if (pool == 1) {
                v = src[i];
            } else {
                float acc = 0.f;
                for (int t = 0; t < len; ++t) acc += src[(long long)t * w + i];
                v = acc / (float)len;  // len == 0 -> NaN, as sum / 0 does in the reference
            }
            ss += v * v;
        }
        vals[j] = v;
    }
    const float nrm = fmaxf(sqrtf(block_sum_256(ss, red)), 1e-12f);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int i = threadIdx.x + 256 * j;
        if (i < w) out[(long long)b * w + i] = normalize ? vals[j] / nrm : vals[j];
    }
}

int bert_head(const float* x, const int32_t* kv_len, int n, int S, int w, int pool, int normalize, float* out,
              cudaStream_t s) {
    if (n <= 0) return 0;
    if (w > 1024) fail(B200_ERR_UNSUPPORTED, "bert_head: width %d > 1024", w);
    bert_head_kernel<<<n, 256, 0, s>>>(x, kv_len, S, w, pool, normalize, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// ------------------------------------------------------------------------------------------------ conversions
__global__ void f32_to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = __float2bfloat16_rn(src[i]);
}
void f32_to_bf16(const float* src, __nv_bfloat16* dst, long long n, cudaStream_t s) {
    if (n <= 0) return;
    f32_to_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(src, dst, n);
    MB_CUDA(cudaGetLastError());
}

__global__ void pad_rows_kernel(const float* __restrict__ src, int rows, int k, int kpad, __nv_bfloat16* __restrict__ dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)rows * kpad) return;
    const int r = (int)(i / kpad), c = (int)(i % kpad);
    dst[i] = __float2bfloat16_rn(c < k ? src[(long long)r * k + c] : 0.f);
}
void pad_rows_to_bf16(const float* src, int rows, int k, int kpad, __nv_bfloat16* dst, cudaStream_t s) {
    const long long n = (long long)rows * kpad;
    pad_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(src, rows, k, kpad, dst);
    MB_CUDA(cudaGetLastError());
}

// conv1.weight [w, 3, p, p] -> the gather GEMM's K order: k' = dy * (64 * kbpd) + dx * 3 + c, zero in the padding slots
__global__ void patch_weight_rows_kernel(const float* __restrict__ src, int rows, int p, int kbpd,
                                         __nv_bfloat16* __restrict__ dst) {
    const int kprime = p * kbpd * 64;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)rows * kprime) return;
    const int r = (int)(i / kprime), k = (int)(i - (long long)r * kprime);
    const int dy = k / (64 * kbpd), q = k - dy * 64 * kbpd;
    float v = 0.f;
    if (q < 3 * p) {
        const int dx = q / 3, c = q - 3 * dx;
        v = src[(long long)r * 3 * p * p + (long long)c * p * p + dy * p + dx];
    }
    dst[i] = __float2bfloat16_rn(v);
}
void patch_weight_rows(const float* src, int rows, int p, int kbpd, __nv_bfloat16* dst, cudaStream_t s) {
    const long long n = (long long)rows * p * kbpd * 64;
    patch_weight_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(src, rows, p, kbpd, dst);
    MB_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ resize
// Pillow's ImagingResample for 8-bit images, restated: per-output-pixel coefficient windows computed in double on
// the host exactly as precompute_coeffs()/normalize_coeffs_8bpc() do (bicubic a = -0.5, support widened by the
// down-scale factor, coefficients rounded to 22-bit fixed point), horizontal pass into an 8-bit intermediate, then
// the vertical pass; each pass accumulates in int32 starting from 1 << 21 and clips (x >> 22) to [0, 255].
constexpr int PRECISION_BITS = 32 - 8 - 2;

struct ResampleTable {
    int ksize = 0;
    std::vector<int> bounds;  // [out][2] = (xmin, xcount)
    std::vector<int> coeffs;  // [out][ksize]
};

static double bicubic_filter(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}

static ResampleTable precompute(int in_size, int out_size) {
    ResampleTable t;
    const double scale = (double)in_size / (double)out_size;
    double filterscale = scale;
    if (filterscale < 1.0) filterscale = 1.0;
    const double support = 2.0 * filterscale;
    t.ksize = (int)ceil(support) * 2 + 1;
    t.bounds.assign((size_t)out_size * 2, 0);
    t.coeffs.assign((size_t)out_size * t.ksize, 0);
    std::vector<double> k(t.ksize);
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = (xx + 0.5) * scale;
        double ww = 0.0;
        const double ss = 1.0 / filterscale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        for (int x = 0; x < xmax; ++x) {
            const double w = bicubic_filter((x + xmin - center + 0.5) * ss);
            k[x] = w;
            ww += w;
        }
        for (int x = 0; x < xmax; ++x)
            if (ww != 0.0) k[x] /= ww;
        for (int x = 0; x < t.ksize; ++x) {
            const double v = x < xmax ? k[x] : 0.0;
            t.coeffs[(size_t)xx * t.ksize + x] =
                v < 0 ? (int)(-0.5 + v * (1 << PRECISION_BITS)) : (int)(0.5 + v * (1 << PRECISION_BITS));
        }
        t.bounds[xx * 2] = xmin;
        t.bounds[xx * 2 + 1] = xmax;
    }
    return t;
}

__device__ __forceinline__ uint8_t clip8(int v) {
    v >>= PRECISION_BITS;
    return (uint8_t)min(max(v, 0), 255);
}

// horizontal: src [n, h, w, 3] -> tmp [n, h, S, 3] for output columns x_off .. x_off + S - 1 of the resized image
__global__ void resample_h_kernel(const uint8_t* __restrict__ src, int n, int h, int w, int S, int x_off,
                                  const int* __restrict__ bounds, const int* __restrict__ coeffs, int ksize,
                                  uint8_t* __restrict__ tmp) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n * h * S) return;
    const int xo = (int)(i % S);
    const long long rowi = i / S;  // (image, y)
    const int xx = xo + x_off;
    const int xmin = bounds[xx * 2], cnt = bounds[xx * 2 + 1];
    const int* k = coeffs + (long long)xx * ksize;
    const uint8_t* line = src + rowi * w * 3;
    int s0 = 1 << (PRECISION_BITS - 1), s1 = s0, s2 = s0;
    for (int x = 0; x < cnt; ++x) {
        const int c = k[x];
        const uint8_t* px = line + (xmin + x) * 3;
        s0 += px[0] * c;
        s1 += px[1] * c;
        s2 += px[2] * c;
    }
    uint8_t* o = tmp + i * 3;
    o[0] = clip8(s0);
    o[1] = clip8(s1);
    o[2] = clip8(s2);
}

// vertical: tmp [n, h, S, 3] -> dst [n, S, S, 3] for output rows y_off .. y_off + S - 1
__global__ void resample_v_kernel(const uint8_t* __restrict__ tmp, int n, int h, int S, int y_off,
                                  const int* __restrict__ bounds, const int* __restrict__ coeffs, int ksize,
                                  uint8_t* __restrict__ dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n * S * S) return;
    const int xo = (int)(i % S);
    const int yo = (int)((i / S) % S);
    const long long b = i / ((long long)S * S);
    const int yy = yo + y_off;
    const int ymin = bounds[yy * 2], cnt = bounds[yy * 2 + 1];
    const int* k = coeffs + (long long)yy * ksize;
    int s0 = 1 << (PRECISION_BITS - 1), s1 = s0, s2 = s0;
    for (int y = 0; y < cnt; ++y) {
        const int c = k[y];
        const uint8_t* px = tmp + ((b * h + ymin + y) * S + xo) * 3;
        s0 += px[0] * c;
        s1 += px[1] * c;
        s2 += px[2] * c;
    }
    uint8_t* o = dst + i * 3;
    o[0] = clip8(s0);
    o[1] = clip8(s1);
    o[2] = clip8(s2);
}

static int py_round_half_even(double v) { return (int)nearbyint(v); }

// Resample [n, h, w, 3] to new_h x new_w and keep the S x S window at (top, left).
static int resample_window_u8(const uint8_t* src, int n, int h, int w, int new_h, int new_w, int top, int left, int S,
                              uint8_t* dst, cudaStream_t s) {
    const ResampleTable th = precompute(w, new_w);
    const ResampleTable tv = precompute(h, new_h);
    {   // stream-ordered temporaries, released on `s` at the end of this block
        auto up = [&](const std::vector<int>& v) {
            DeviceBuffer<int> d(v.size(), s);
            MB_CUDA(cudaMemcpyAsync(d.get(), v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice, s));
            return d;
        };
        const DeviceBuffer<int> d_hb = up(th.bounds), d_hc = up(th.coeffs), d_vb = up(tv.bounds), d_vc = up(tv.coeffs);
        const DeviceBuffer<uint8_t> tmp((size_t)n * h * S * 3, s);
        const long long nh = (long long)n * h * S;
        resample_h_kernel<<<(unsigned)((nh + 255) / 256), 256, 0, s>>>(src, n, h, w, S, left, d_hb.get(), d_hc.get(),
                                                                       th.ksize, tmp.get());
        MB_CUDA(cudaGetLastError());
        const long long nv = (long long)n * S * S;
        resample_v_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, s>>>(tmp.get(), n, h, S, top, d_vb.get(), d_vc.get(),
                                                                       tv.ksize, dst);
        MB_CUDA(cudaGetLastError());
    }
    // the pageable host vectors above must outlive the async copies: synchronise before they go out of scope
    MB_CUDA(cudaStreamSynchronize(s));
    return 2;
}

int resize_crop_u8(const uint8_t* src, int n, int h, int w, int S, uint8_t* dst, cudaStream_t s) {
    if (n <= 0) return 0;
    // torchvision Resize(S): shortest side -> S, the other int(S * long / short); CenterCrop(S)
    int new_w, new_h;
    if (w <= h) {
        new_w = S;
        new_h = (int)((double)((long long)S * h) / (double)w);  // int(S * long / short): Python true division
    } else {
        new_h = S;
        new_w = (int)((double)((long long)S * w) / (double)h);
    }
    const int left = py_round_half_even((new_w - S) / 2.0);
    const int top = py_round_half_even((new_h - S) / 2.0);
    return resample_window_u8(src, n, h, w, new_h, new_w, top, left, S, dst, s);
}

int resize_squash_u8(const uint8_t* src, int n, int h, int w, int S, uint8_t* dst, cudaStream_t s) {
    if (n <= 0) return 0;
    // PIL resize((S, S), BICUBIC) = torchvision Resize((S, S)) on a PIL image: both axes to S, nothing cropped.  An axis
    // that already has S pixels gets the identity coefficients (a single 1.0 tap), so running its pass is exact.
    return resample_window_u8(src, n, h, w, S, S, 0, 0, S, dst, s);
}

// ------------------------------------------------------------------------------------------------ SigLIP MAP head
// One CTA (128 threads) per (image, head).  Pass 1: thread s takes key s (its 64 bf16 values are one 128-byte line)
// and stores the base-2 logit q.k / 8 * log2(e) in shared memory; pass 2: block max, p = exp2(l - max) in place, block
// sum; pass 3: warp w accumulates p_s v_s over keys s = w (mod 4), lane l owning columns 2l, 2l + 1; the four partial
// sums are added in a fixed order and divided by the sum.  Two exact passes over the logits instead of an online
// softmax: S <= MAP_MAX_TOKENS logits fit in shared memory.
constexpr int MAP_THREADS = 128;
constexpr int MAP_MAX_TOKENS = 12288;   // 48 KB of logits

__device__ __forceinline__ float block_reduce_128(float v, float* red, bool is_max) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float u = __shfl_xor_sync(0xffffffffu, v, o);
        v = is_max ? fmaxf(v, u) : v + u;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();   // red[] may still be read by the previous reduction
    if (lane == 0) red[warp] = v;
    __syncthreads();
    return is_max ? fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3])) : ((red[0] + red[1]) + red[2]) + red[3];
}

__global__ void __launch_bounds__(MAP_THREADS) map_attention_kernel(const float* __restrict__ q, long long q_stride,
                                                                    const __nv_bfloat16* __restrict__ kv, int S, int W,
                                                                    __nv_bfloat16* __restrict__ out) {
    extern __shared__ float logit[];   // [S]
    __shared__ float qs[64];
    __shared__ float red[4];
    __shared__ float part[4][64];
    const int b = blockIdx.x, h = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid < 64) qs[tid] = q[b * q_stride + h * 64 + tid] * (0.125f * 1.4426950408889634f);
    __syncthreads();
    const long long ld = 2LL * W;
    const __nv_bfloat16* keys = kv + (long long)b * S * ld + h * 64;
    const __nv_bfloat16* vals = keys + W;
    float mx = -INFINITY;
    for (int s = tid; s < S; s += MAP_THREADS) {
        const uint4* k4 = reinterpret_cast<const uint4*>(keys + s * ld);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint4 u = __ldg(k4 + j);
            const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __bfloat1622float2(p2[e]);
                acc = fmaf(qs[8 * j + 2 * e], f.x, acc);
                acc = fmaf(qs[8 * j + 2 * e + 1], f.y, acc);
            }
        }
        logit[s] = acc;
        mx = fmaxf(mx, acc);
    }
    mx = block_reduce_128(mx, red, true);
    float sum = 0.f;
    for (int s = tid; s < S; s += MAP_THREADS) {
        const float p = exp2f(logit[s] - mx);
        logit[s] = p;
        sum += p;
    }
    sum = block_reduce_128(sum, red, false);   // its barriers also publish the p values
    float2 acc = make_float2(0.f, 0.f);
    for (int s = warp; s < S; s += 4) {
        const float p = logit[s];
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(vals + s * ld + 2 * lane));
        acc.x = fmaf(p, f.x, acc.x);
        acc.y = fmaf(p, f.y, acc.y);
    }
    part[warp][2 * lane] = acc.x;
    part[warp][2 * lane + 1] = acc.y;
    __syncthreads();
    if (tid < 64) {
        const float o = ((part[0][tid] + part[1][tid]) + part[2][tid]) + part[3][tid];
        out[(long long)b * W + h * 64 + tid] = __float2bfloat16_rn(o / sum);
    }
}

int map_attention(const float* q, long long q_stride, const __nv_bfloat16* kv, int n, int S, int W, int heads,
                  __nv_bfloat16* out, cudaStream_t s) {
    if (n <= 0) return 0;
    if (W != heads * 64) fail(B200_ERR_UNSUPPORTED, "map_attention: head_dim must be 64 (width %d, heads %d)", W, heads);
    if (S <= 0 || S > MAP_MAX_TOKENS) fail(B200_ERR_UNSUPPORTED, "map_attention: %d tokens (1..%d)", S, MAP_MAX_TOKENS);
    map_attention_kernel<<<dim3((unsigned)n, (unsigned)heads), MAP_THREADS, (size_t)S * sizeof(float), s>>>(
        q, q_stride, kv, S, W, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// ------------------------------------------------------------------------------------------------ ResNet trunk
// One thread = 8 consecutive k of one output pixel: k = tap * 3 + c (tap = 3 ky + kx), zero for k >= 27.  Input pixel
// (2 oy - 1 + ky, 2 ox - 1 + kx), zero outside the image: the convolution pads the normalised image.
__global__ void __launch_bounds__(256) stem_im2col_kernel(const uint8_t* __restrict__ u8, const float* __restrict__ chw,
                                                          int n, int S, float3 nscale, float3 nshift,
                                                          __nv_bfloat16* __restrict__ out) {
    const int So = S / 2;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)n * So * So * 8;
    if (gid >= total) return;
    const int kg = (int)(gid & 7);
    const long long pix = gid >> 3;
    const long long b = pix / ((long long)So * So);
    const int rem = (int)(pix - b * So * So), oy = rem / So, ox = rem - oy * So;
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int k = kg * 8 + e, tap = k / 3, c = k - tap * 3;
        const int iy = 2 * oy - 1 + tap / 3, ix = 2 * ox - 1 + tap % 3;
        float v = 0.f;
        if (k < 27 && (unsigned)iy < (unsigned)S && (unsigned)ix < (unsigned)S) {
            if (u8 != nullptr) {
                const float sc = c == 0 ? nscale.x : c == 1 ? nscale.y : nscale.z;
                const float sh = c == 0 ? nshift.x : c == 1 ? nshift.y : nshift.z;
                v = fmaf((float)__ldg(u8 + ((b * S + iy) * S + ix) * 3 + c), sc, sh);
            } else {
                v = __ldg(chw + ((b * 3 + c) * S + iy) * S + ix);
            }
        }
        f[e] = v;
    }
    reinterpret_cast<uint4*>(out)[gid] =
        make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

int stem_im2col(const uint8_t* u8, const float* chw, int n, int S, const float* mean, const float* std,
                __nv_bfloat16* out, cudaStream_t s) {
    if (n <= 0) return 0;
    if (S % 2 != 0) fail(B200_ERR_INTERNAL, "stem_im2col: image size %d must be even", S);
    float sc[3], sh[3];
    for (int c = 0; c < 3; ++c) {   // the patch gather's constants (gemm.cu launch_tiles)
        sc[c] = (float)(1.0 / (255.0 * (double)std[c]));
        sh[c] = (float)(-(double)mean[c] / (double)std[c]);
    }
    const long long total = (long long)n * (S / 2) * (S / 2) * 8;
    stem_im2col_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(u8, chw, n, S, make_float3(sc[0], sc[1], sc[2]),
                                                                        make_float3(sh[0], sh[1], sh[2]), out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// One thread = 8 channels of one output pixel; the four inputs are summed in fp32 and scaled by 1/4.
__global__ void __launch_bounds__(256) avgpool2_kernel(const uint4* __restrict__ in, int n, int H, int W, int C8,
                                                       uint4* __restrict__ out) {
    const int Ho = H / 2, Wo = W / 2;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)n * Ho * Wo * C8;
    if (gid >= total) return;
    const int c = (int)(gid % C8);
    const long long pix = gid / C8;
    const long long b = pix / ((long long)Ho * Wo);
    const int rem = (int)(pix - b * Ho * Wo), oy = rem / Wo, ox = rem - oy * Wo;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int d = 0; d < 4; ++d) {
        const uint4 u = __ldg(in + ((b * H + 2 * oy + (d >> 1)) * W + 2 * ox + (d & 1)) * C8 + c);
        const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __bfloat1622float2(p2[e]);
            acc[2 * e] += f.x;
            acc[2 * e + 1] += f.y;
        }
    }
    out[gid] = make_uint4(pack_bf16x2(0.25f * acc[0], 0.25f * acc[1]), pack_bf16x2(0.25f * acc[2], 0.25f * acc[3]),
                          pack_bf16x2(0.25f * acc[4], 0.25f * acc[5]), pack_bf16x2(0.25f * acc[6], 0.25f * acc[7]));
}

int avgpool2_nhwc(const __nv_bfloat16* in, int n, int H, int W, int C, __nv_bfloat16* out, cudaStream_t s) {
    if (n <= 0) return 0;
    if (H % 2 != 0 || W % 2 != 0 || C % 8 != 0) fail(B200_ERR_INTERNAL, "avgpool2: %d x %d x %d", H, W, C);
    const long long total = (long long)n * (H / 2) * (W / 2) * (C / 8);
    avgpool2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(reinterpret_cast<const uint4*>(in), n, H, W, C / 8,
                                                                     reinterpret_cast<uint4*>(out));
    MB_CUDA(cudaGetLastError());
    return 1;
}

// One thread = 8 channels of one image: the fp32 mean over the HW pixels, then every token row.
__global__ void __launch_bounds__(256) attnpool_tokens_kernel(const uint4* __restrict__ x, const float4* __restrict__ pos,
                                                              int n, int HW, int C8, uint4* __restrict__ out) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)n * C8) return;
    const int c = (int)(gid % C8);
    const long long b = gid / C8;
    const uint4* src = x + b * HW * C8 + c;
    uint4* dst = out + b * (HW + 1) * C8 + c;
    float mean[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < HW; ++s) {
        const uint4 u = __ldg(src + (long long)s * C8);
        const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&u);
        const float4 p0 = __ldg(pos + (long long)(1 + s) * 2 * C8 + 2 * c), p1 = __ldg(pos + (long long)(1 + s) * 2 * C8 + 2 * c + 1);
        const float pv[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
        float v[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __bfloat1622float2(p2[e]);
            mean[2 * e] += f.x;
            mean[2 * e + 1] += f.y;
            v[2 * e] = f.x + pv[2 * e];
            v[2 * e + 1] = f.y + pv[2 * e + 1];
        }
        dst[(long long)(1 + s) * C8] = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                                                  pack_bf16x2(v[6], v[7]));
    }
    const float4 p0 = __ldg(pos + 2 * c), p1 = __ldg(pos + 2 * c + 1);
    const float pv[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = mean[e] / (float)HW + pv[e];
    dst[0] = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

int attnpool_tokens(const __nv_bfloat16* x, const float* pos, int n, int HW, int C, __nv_bfloat16* out, cudaStream_t s) {
    if (n <= 0) return 0;
    if (C % 8 != 0) fail(B200_ERR_INTERNAL, "attnpool_tokens: C = %d must be a multiple of 8", C);
    const long long total = (long long)n * (C / 8);
    attnpool_tokens_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
        reinterpret_cast<const uint4*>(x), reinterpret_cast<const float4*>(pos), n, HW, C / 8, reinterpret_cast<uint4*>(out));
    MB_CUDA(cudaGetLastError());
    return 1;
}

__global__ void __launch_bounds__(256) l2_rows_kernel(const float* __restrict__ src, int n, int E, int normalize,
                                                      float* __restrict__ out) {
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= n) return;
    const float* row = src + (long long)b * E;
    float ss = 0.f;
    if (normalize)
        for (int i = lane; i < E; i += 32) ss += row[i] * row[i];
    const float nrm = sqrtf(warp_sum(ss));
    for (int i = lane; i < E; i += 32) out[(long long)b * E + i] = normalize ? row[i] / nrm : row[i];
}

int l2_rows(const float* src, int n, int E, int normalize, float* out, cudaStream_t s) {
    if (n <= 0) return 0;
    l2_rows_kernel<<<(n + 7) / 8, 256, 0, s>>>(src, n, E, normalize, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// ------------------------------------------------------------------------------------------------ ConvNeXt
// The image tower's memory-bound kernels over fp32 NHWC pixel rows x [pixels, C] (C % 64 == 0, C <= 3072).  A CTA has
// one thread per 4 channels (rounded up to whole warps) and holds P pixels of them in registers; pixel_ln normalises
// each pixel over its C channels (fp32 statistics, mean then variance, as layernorm_kernel does).
constexpr int PX_MAX_C = 3072;

static int px_threads(int C) { return (C / 4 + 31) / 32 * 32; }

// v[p] (this thread's 4 channels of pixel p; zeros when !active) -> LayerNorm(pixel p) * gamma + beta.  red: shared
// scratch of 32 * P floats.  Every thread of the CTA must call it.
template <int P>
__device__ __forceinline__ void pixel_ln(float4 (&v)[P], bool active, int C, const float* __restrict__ gamma,
                                         const float* __restrict__ beta, float eps, float* red) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    float mean[P], rstd[P];
#pragma unroll
    for (int p = 0; p < P; ++p) {
        const float s = warp_sum(v[p].x + v[p].y + v[p].z + v[p].w);
        if (lane == 0) red[warp * P + p] = s;
    }
    __syncthreads();
#pragma unroll
    for (int p = 0; p < P; ++p) {
        float s = 0.f;
        for (int i = 0; i < nwarps; ++i) s += red[i * P + p];
        mean[p] = s / (float)C;
    }
    __syncthreads();
#pragma unroll
    for (int p = 0; p < P; ++p) {
        const float a = v[p].x - mean[p], b = v[p].y - mean[p], c = v[p].z - mean[p], d = v[p].w - mean[p];
        const float q = warp_sum(active ? a * a + b * b + c * c + d * d : 0.f);
        if (lane == 0) red[warp * P + p] = q;
    }
    __syncthreads();
#pragma unroll
    for (int p = 0; p < P; ++p) {
        float q = 0.f;
        for (int i = 0; i < nwarps; ++i) q += red[i * P + p];
        rstd[p] = 1.0f / sqrtf(q / (float)C + eps);
    }
    if (!active) return;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + threadIdx.x);
    const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + threadIdx.x);
#pragma unroll
    for (int p = 0; p < P; ++p) {
        v[p].x = (v[p].x - mean[p]) * rstd[p] * g.x + b.x;
        v[p].y = (v[p].y - mean[p]) * rstd[p] * g.y + b.y;
        v[p].z = (v[p].z - mean[p]) * rstd[p] * g.z + b.z;
        v[p].w = (v[p].w - mean[p]) * rstd[p] * g.w + b.w;
    }
}

__device__ __forceinline__ uint2 pack_bf16x4(const float4& y) {
    return make_uint2(pack_bf16x2(y.x, y.y), pack_bf16x2(y.z, y.w));
}

__device__ __forceinline__ void fma4(float4& acc, const float4& w, const float4& x) {
    acc.x = fmaf(w.x, x.x, acc.x);
    acc.y = fmaf(w.y, x.y, acc.y);
    acc.z = fmaf(w.z, x.z, acc.z);
    acc.w = fmaf(w.w, x.w, acc.w);
}

// 7 x 7 depthwise conv (zero padding 3) + bias, then LayerNorm over C, of P consecutive pixels of one image row:
// x fp32 [n, H, W, C], w fp32 [49, C] (tap-major), out bf16 [n * H * W, C].  Along a row the 7 taps slide over the
// P + 6 input pixels in registers, so each input row is loaded once per output row (the other six output rows that
// read it find it in L1 / L2); the conv result never leaves registers.
template <int P>
__global__ void __launch_bounds__(P == 8 ? 256 : 768, P == 8 ? 2 : 1) dwconv7_ln_kernel(
    const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
    const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int H, int W, int C, int xtiles,
    __nv_bfloat16* __restrict__ out) {
    __shared__ float red[32 * P];
    const int xt = blockIdx.x % xtiles;
    const long long row = blockIdx.x / xtiles;   // b * H + y
    const int y = (int)(row % H), x0 = xt * P, C4 = C / 4, c4 = threadIdx.x;
    const bool active = c4 < C4;
    const long long img = row - y;               // b * H
    float4 acc[P];
    const float4 b4 = active ? __ldg(reinterpret_cast<const float4*>(bias) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int p = 0; p < P; ++p) acc[p] = b4;
    if (active) {
        const float4* w4 = reinterpret_cast<const float4*>(w) + c4;
        for (int dy = 0; dy < 7; ++dy) {
            const int yy = y + dy - 3;
            if (yy < 0 || yy >= H) continue;
            const float4* src = reinterpret_cast<const float4*>(x) + (img + yy) * W * C4 + c4;
            float4 wt[7];
#pragma unroll
            for (int dx = 0; dx < 7; ++dx) wt[dx] = __ldg(w4 + (dy * 7 + dx) * C4);
#pragma unroll
            for (int j = 0; j < P + 6; ++j) {
                const int xx = x0 + j - 3;
                const float4 in = xx >= 0 && xx < W ? __ldg(src + (long long)xx * C4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int p = 0; p < P; ++p)
                    if (j - p >= 0 && j - p < 7) fma4(acc[p], wt[j - p], in);
            }
        }
    }
    // (pixels past the row end take part in the reductions but are not written)
    pixel_ln<P>(acc, active, C, gamma, beta, eps, red);
    if (!active) return;
    uint2* o = reinterpret_cast<uint2*>(out) + (row * W + x0) * C4 + c4;
#pragma unroll
    for (int p = 0; p < P; ++p)
        if (x0 + p < W) o[(long long)p * C4] = pack_bf16x4(acc[p]);
}

static void check_px_width(int C) {
    if (C <= 0 || C % 64 != 0 || C > PX_MAX_C)
        fail(B200_ERR_UNSUPPORTED, "ConvNeXt: %d channels (a multiple of 64, <= %d, is needed)", C, PX_MAX_C);
}

int dwconv7_ln(const float* x, int n, int H, int W, int C, const float* w49, const float* bias, const float* gamma,
               const float* beta, float eps, __nv_bfloat16* out, cudaStream_t s) {
    if (n <= 0) return 0;
    check_px_width(C);
    // 8 pixels per thread up to 1024 channels (256 threads); 4 above, to stay within 80 registers at 768 threads
    if (C <= 1024) {
        const int xtiles = (W + 7) / 8;
        dwconv7_ln_kernel<8><<<(unsigned)((long long)n * H * xtiles), px_threads(C), 0, s>>>(x, w49, bias, gamma, beta,
                                                                                             eps, H, W, C, xtiles, out);
    } else {
        const int xtiles = (W + 3) / 4;
        dwconv7_ln_kernel<4><<<(unsigned)((long long)n * H * xtiles), px_threads(C), 0, s>>>(x, w49, bias, gamma, beta,
                                                                                             eps, H, W, C, xtiles, out);
    }
    MB_CUDA(cudaGetLastError());
    return 1;
}

// LayerNorm over C of LNP_P consecutive pixels of x fp32 [n, H, W, C] per CTA.  PATCHIFY: bf16 into the 2 x 2 stride-2
// downsample's GEMM rows, pixel (b, y, x) -> row (b, y/2, x/2), columns ((y % 2) * 2 + x % 2) * C + c; otherwise fp32
// back to the same pixel row (out may be x).
constexpr int LNP_P = 4;

template <bool PATCHIFY>
__global__ void __launch_bounds__(768) ln_pixels_kernel(const float* x, long long pixels, int H, int W, int C,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        float eps, void* out) {
    __shared__ float red[32 * LNP_P];
    const int C4 = C / 4, c4 = threadIdx.x;
    const bool active = c4 < C4;
    const long long p0 = (long long)blockIdx.x * LNP_P;
    float4 v[LNP_P];
#pragma unroll
    for (int p = 0; p < LNP_P; ++p)
        v[p] = active && p0 + p < pixels ? reinterpret_cast<const float4*>(x)[(p0 + p) * C4 + c4]
                                         : make_float4(0.f, 0.f, 0.f, 0.f);
    pixel_ln<LNP_P>(v, active, C, gamma, beta, eps, red);
    if (!active) return;
#pragma unroll
    for (int p = 0; p < LNP_P; ++p) {
        const long long r = p0 + p;
        if (r >= pixels) break;
        if (PATCHIFY) {
            const int xx = (int)(r % W);
            const long long by = r / W;
            const int yy = (int)(by % H);
            const long long b = by / H;
            const long long orow = (b * (H / 2) + yy / 2) * (W / 2) + xx / 2;
            const int q = (yy & 1) * 2 + (xx & 1);
            reinterpret_cast<uint2*>(out)[orow * C + (long long)q * C4 + c4] = pack_bf16x4(v[p]);
        } else {
            reinterpret_cast<float4*>(out)[r * C4 + c4] = v[p];
        }
    }
}

int ln_pixels(const float* x, int n, int H, int W, int C, const float* gamma, const float* beta, float eps,
              float* out_f32, __nv_bfloat16* out_patch, cudaStream_t s) {
    if (n <= 0) return 0;
    check_px_width(C);
    if ((out_f32 != nullptr) == (out_patch != nullptr)) fail(B200_ERR_INTERNAL, "ln_pixels: exactly one output");
    if (out_patch && (H % 2 != 0 || W % 2 != 0)) fail(B200_ERR_INTERNAL, "ln_pixels: %d x %d is not even", H, W);
    const long long pixels = (long long)n * H * W;
    const unsigned grid = (unsigned)((pixels + LNP_P - 1) / LNP_P);
    if (out_patch)
        ln_pixels_kernel<true><<<grid, px_threads(C), 0, s>>>(x, pixels, H, W, C, gamma, beta, eps, out_patch);
    else
        ln_pixels_kernel<false><<<grid, px_threads(C), 0, s>>>(x, pixels, H, W, C, gamma, beta, eps, out_f32);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// Global average pool of each image's HW pixel rows of x fp32 [n, HW, C], then LayerNorm over C -> bf16 [n, C] (the
// head GEMM's A operand): one CTA per image.
__global__ void __launch_bounds__(768) pool_ln_kernel(const float* __restrict__ x, int HW, int C,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      float eps, __nv_bfloat16* __restrict__ out) {
    __shared__ float red[32];
    const int C4 = C / 4, c4 = threadIdx.x;
    const bool active = c4 < C4;
    float4 v[1] = {make_float4(0.f, 0.f, 0.f, 0.f)};
    if (active) {
        const float4* src = reinterpret_cast<const float4*>(x) + (long long)blockIdx.x * HW * C4 + c4;
        for (int i = 0; i < HW; ++i) {
            const float4 a = __ldg(src + (long long)i * C4);
            v[0].x += a.x;
            v[0].y += a.y;
            v[0].z += a.z;
            v[0].w += a.w;
        }
        const float inv = 1.0f / (float)HW;
        v[0] = make_float4(v[0].x * inv, v[0].y * inv, v[0].z * inv, v[0].w * inv);
    }
    pixel_ln<1>(v, active, C, gamma, beta, eps, red);
    if (active) reinterpret_cast<uint2*>(out)[(long long)blockIdx.x * C4 + c4] = pack_bf16x4(v[0]);
}

int pool_ln(const float* x, int n, int HW, int C, const float* gamma, const float* beta, float eps, __nv_bfloat16* out,
            cudaStream_t s) {
    if (n <= 0) return 0;
    check_px_width(C);
    if (HW <= 0) fail(B200_ERR_INTERNAL, "pool_ln: %d pixels", HW);
    pool_ln_kernel<<<n, px_threads(C), 0, s>>>(x, HW, C, gamma, beta, eps, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace kernels
}  // namespace mb
