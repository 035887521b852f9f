#include "kernels.cuh"

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
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

// CLS (CoCa's text tower): ids are [n, S - 1]; row s < S - 1 of a sequence is tok[ids[s]] + pos[s], its last row
// cls + pos[S - 1], and the pooled row eot is S - 1.
template <bool CLS>
__global__ void __launch_bounds__(256) clip_text_embed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ tok,
                                                              const float* __restrict__ pos, int n, int S, int w, int vocab,
                                                              float* __restrict__ x, int32_t* __restrict__ eot,
                                                              const float* __restrict__ cls) {
    // one warp per token row
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= (long long)n * S) return;
    const int s = (int)(row % S);
    if constexpr (CLS) {
        const long long b = row / S;
        const float* src = cls;
        if (s < S - 1) {
            const int id = min(max(ids[b * (S - 1) + s], 0), vocab - 1);
            src = tok + (long long)id * w;
        }
        const float4* t4 = reinterpret_cast<const float4*>(src);
        const float4* p4 = reinterpret_cast<const float4*>(pos + (long long)s * w);
        float4* o4 = reinterpret_cast<float4*>(x + row * w);
        for (int i = lane; i < w / 4; i += 32) {
            const float4 a = __ldg(t4 + i), c = __ldg(p4 + i);
            o4[i] = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);
        }
        if (s == 0 && lane == 0) eot[b] = S - 1;
        return;
    }
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
                    int32_t* eot, cudaStream_t s, const float* cls) {
    if (n <= 0) return 0;
    const long long rows = (long long)n * S;
    const unsigned blocks = (unsigned)((rows + 7) / 8);
    if (cls)
        clip_text_embed_kernel<true><<<blocks, 256, 0, s>>>(ids, tok, pos, n, S, w, vocab, x, eot, cls);
    else
        clip_text_embed_kernel<false><<<blocks, 256, 0, s>>>(ids, tok, pos, n, S, w, vocab, x, eot, nullptr);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// POS: BERT's position_embeddings row s is added; GTE (NewModel, rotary positions) has no position table.
// TYPES: each token adds row type_ids[row] (clamped to [0, type_vocab - 1]) of the token-type table `type0`
// [type_vocab, w] (a sentence pair); without it every token adds row 0, and the instantiation is the one the encoders
// have always run.
template <bool POS, bool TYPES = false>
__global__ void __launch_bounds__(256) bert_embed_ln_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ mask,
                                                            const float* __restrict__ word, const float* __restrict__ pos,
                                                            const float* __restrict__ type0, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float eps, int n, int S, int w,
                                                            int vocab, float* __restrict__ x, __nv_bfloat16* __restrict__ h,
                                                            int32_t* __restrict__ kv_len,
                                                            const int32_t* __restrict__ type_ids = nullptr,
                                                            int type_vocab = 1) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= (long long)n * S) return;
    const int s = (int)(row % S);
    int id = ids[row];
    id = min(max(id, 0), vocab - 1);
    const int nv = w / 128;
    const float4* w4 = reinterpret_cast<const float4*>(word + (long long)id * w);
    const float* trow = type0;
    if constexpr (TYPES) trow += (long long)min(max(type_ids[row], 0), type_vocab - 1) * w;
    const float4* t4 = reinterpret_cast<const float4*>(trow);
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
                  __nv_bfloat16* h, int32_t* kv_len, cudaStream_t s, const int32_t* type_ids, int type_vocab) {
    if (n <= 0) return 0;
    check_ln_width(w);
    const long long rows = (long long)n * S;
    const unsigned blocks = (unsigned)((rows + 7) / 8);
    if (type_ids) {
        if (!pos || type_vocab < 1) fail(B200_ERR_INTERNAL, "bert_embed_ln: token types need positions and a table");
        bert_embed_ln_kernel<true, true><<<blocks, 256, 0, s>>>(ids, mask, word, pos, type0, gamma, beta, eps, n, S, w,
                                                                 vocab, x, h, kv_len, type_ids, type_vocab);
    } else if (pos)
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

// bias (fp32 [E], NULL: none) is added after the four K-slices are summed
__global__ void __launch_bounds__(256) head_proj_kernel(const float* __restrict__ pooled, const float* __restrict__ proj,
                                                        const float* __restrict__ bias, int n, int w, int E,
                                                        float* __restrict__ out) {
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
                const float v = ((part[0][k][c] + part[1][k][c]) + part[2][k][c]) + part[3][k][c];
                out[(long long)(b0 + k) * E + e] = bias ? v + bias[e] : v;
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

// CoCa's encode_image / encode_text (normalize=True, their default): F.normalize (x / max(|x|, 1e-12)), then, when
// normalize is set, Marqo's own division by the norm (no epsilon) of the already unit row.
__global__ void __launch_bounds__(256) head_unit_kernel(float* __restrict__ out, int n, int E, int normalize) {
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= n) return;
    float* row = out + (long long)b * E;
    float ss = 0.f;
    for (int i = lane; i < E; i += 32) ss += row[i] * row[i];
    const float den = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
    ss = 0.f;
    for (int i = lane; i < E; i += 32) {
        const float v = row[i] / den;
        row[i] = v;
        ss += v * v;
    }
    if (!normalize) return;
    const float nrm = sqrtf(warp_sum(ss));
    for (int i = lane; i < E; i += 32) row[i] = row[i] / nrm;
}

int clip_head(const float* x, int S, const int32_t* row_in_seq, const float* gamma, const float* beta, float eps,
              const float* proj, int n, int w, int E, int normalize, float* out, float* pooled_ws, cudaStream_t s,
              bool unit) {
    if (n <= 0) return 0;
    if (w % 4 != 0 || (size_t)HEAD_IMGS * w * sizeof(float) > 40 * 1024)
        fail(B200_ERR_UNSUPPORTED, "clip_head: width %d unsupported", w);
    head_ln_kernel<<<(n + 7) / 8, 256, 0, s>>>(x, S, row_in_seq, gamma, beta, eps, n, w, pooled_ws);
    MB_CUDA(cudaGetLastError());
    const dim3 grid((n + HEAD_IMGS - 1) / HEAD_IMGS, (E + HEAD_COLS - 1) / HEAD_COLS);
    head_proj_kernel<<<grid, 256, (size_t)HEAD_IMGS * w * sizeof(float), s>>>(pooled_ws, proj, nullptr, n, w, E, out);
    MB_CUDA(cudaGetLastError());
    if (unit) {
        head_unit_kernel<<<(n + 7) / 8, 256, 0, s>>>(out, n, E, normalize);
        MB_CUDA(cudaGetLastError());
        return 3;
    }
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

int text_head(const float* x, const int32_t* kv_len, int n, int S, int w, const float* proj, const float* bias, int E,
              int normalize, float* out, float* pooled_ws, cudaStream_t s) {
    if (n <= 0) return 0;
    if (w > 1024 || w % 4 != 0) fail(B200_ERR_UNSUPPORTED, "text_head: width %d unsupported", w);
    bert_head_kernel<<<n, 256, 0, s>>>(x, kv_len, S, w, 0, 0, pooled_ws);
    MB_CUDA(cudaGetLastError());
    const dim3 grid((n + HEAD_IMGS - 1) / HEAD_IMGS, (E + HEAD_COLS - 1) / HEAD_COLS);
    head_proj_kernel<<<grid, 256, (size_t)HEAD_IMGS * w * sizeof(float), s>>>(pooled_ws, proj, bias, n, w, E, out);
    MB_CUDA(cudaGetLastError());
    if (!normalize) return 2;
    head_norm_kernel<<<(n + 7) / 8, 256, 0, s>>>(out, n, E);
    MB_CUDA(cudaGetLastError());
    return 3;
}

// BertForSequenceClassification's head, CLS_SEQS sequences per CTA so that each pooler row is read once per CTA: the
// CLS rows in shared memory, one warp per pooler output (every warp's lanes stride over a coalesced weight row, then a
// butterfly sum: a fixed order), tanh, then one warp per (sequence, label) for the classifier.  Everything is fp32.
constexpr int CLS_SEQS = 4;

__global__ void __launch_bounds__(256) cls_head_kernel(const float* __restrict__ x, int S, int n, int w,
                                                       const float* __restrict__ wp, const float* __restrict__ bp,
                                                       const float* __restrict__ wc, const float* __restrict__ bc, int L,
                                                       int sigmoid, float* __restrict__ out) {
    extern __shared__ float sm[];   // cls [CLS_SEQS][w], then pooled [CLS_SEQS][w]
    float* cls = sm;
    float* pooled = sm + CLS_SEQS * w;
    const int b0 = blockIdx.x * CLS_SEQS, nb = min(CLS_SEQS, n - b0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < CLS_SEQS * w; i += 256) {
        const int k = i / w, c = i - k * w;
        cls[i] = k < nb ? x[(long long)(b0 + k) * S * w + c] : 0.f;   // token 0 of sequence b0 + k
    }
    __syncthreads();
    for (int o = warp; o < w; o += 8) {
        const float* row = wp + (long long)o * w;
        float acc[CLS_SEQS];
#pragma unroll
        for (int k = 0; k < CLS_SEQS; ++k) acc[k] = 0.f;
        for (int i = lane; i < w; i += 32) {
            const float a = __ldg(row + i);
#pragma unroll
            for (int k = 0; k < CLS_SEQS; ++k) acc[k] = fmaf(a, cls[k * w + i], acc[k]);
        }
#pragma unroll
        for (int k = 0; k < CLS_SEQS; ++k) {
            const float v = warp_sum(acc[k]);
            if (lane == 0) pooled[k * w + o] = tanhf(v + bp[o]);
        }
    }
    __syncthreads();
    for (int j = warp; j < nb * L; j += 8) {
        const int k = j / L, l = j - k * L;
        const float* row = wc + (long long)l * w;
        float acc = 0.f;
        for (int i = lane; i < w; i += 32) acc = fmaf(__ldg(row + i), pooled[k * w + i], acc);
        acc = warp_sum(acc) + bc[l];
        if (lane == 0) out[(long long)(b0 + k) * L + l] = sigmoid ? 1.f / (1.f + expf(-acc)) : acc;
    }
}

int cls_head(const float* x, int S, int n, int w, const float* wp, const float* bp, const float* wc, const float* bc,
             int L, int sigmoid, float* out, cudaStream_t s) {
    if (n <= 0) return 0;
    if (w <= 0 || w > 1024 || L <= 0) fail(B200_ERR_UNSUPPORTED, "cls_head: width %d, %d labels unsupported", w, L);
    const size_t smem = (size_t)2 * CLS_SEQS * w * sizeof(float);   // <= 32 KB
    cls_head_kernel<<<(n + CLS_SEQS - 1) / CLS_SEQS, 256, smem, s>>>(x, S, n, w, wp, bp, wc, bc, L, sigmoid, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// ------------------------------------------------------------------------------------------------ OWL-ViT head
// A row in registers (lane holds float4 j at column 4 (lane + 32 j)) normalised in place: ln_row's arithmetic.
__device__ __forceinline__ void ln_regs(float4 (&v)[LN_MAX_V4], int nv, int w, const float* gamma, const float* beta,
                                        float eps, int lane) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < LN_MAX_V4; ++j)
        if (j < nv) s += v[j].x + v[j].y + v[j].z + v[j].w;
    const float mean = warp_sum(s) / (float)w;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < LN_MAX_V4; ++j)
        if (j < nv) {
            const float a = v[j].x - mean, b = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
            q += a * a + b * b + c * c + d * d;
        }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)w + eps);
#pragma unroll
    for (int j = 0; j < LN_MAX_V4; ++j)
        if (j < nv) {
            const int i4 = lane + 32 * j;
            const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + i4);
            const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + i4);
            v[j].x = (v[j].x - mean) * rstd * g.x + b.x;
            v[j].y = (v[j].y - mean) * rstd * g.y + b.y;
            v[j].z = (v[j].z - mean) * rstd * g.z + b.z;
            v[j].w = (v[j].w - mean) * rstd * g.w + b.w;
        }
}

// One warp per patch row: the class row and the patch row through ln_post (the class row's LayerNorm is recomputed
// by every warp of its image: one L2-resident row, cheaper than a second launch), their product through the
// detector's LayerNorm, written as bf16 for the head GEMMs.
__global__ void __launch_bounds__(256) owl_merge_ln_kernel(const float* __restrict__ x, int n, int N, int w,
                                                           const float* __restrict__ post_g,
                                                           const float* __restrict__ post_b,
                                                           const float* __restrict__ det_g,
                                                           const float* __restrict__ det_b, float eps,
                                                           __nv_bfloat16* __restrict__ out) {
    const int P = N - 1;
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= (long long)n * P) return;
    const long long b = row / P, p = row - b * P + 1;
    const int nv = w / 128;
    const float* cls = x + b * N * w;
    const float* pat = cls + p * w;
    float4 c[LN_MAX_V4], v[LN_MAX_V4];
#pragma unroll
    for (int j = 0; j < LN_MAX_V4; ++j)
        if (j < nv) {
            c[j] = load4(cls, lane + 32 * j);
            v[j] = load4(pat, lane + 32 * j);
        }
    ln_regs(c, nv, w, post_g, post_b, eps, lane);
    ln_regs(v, nv, w, post_g, post_b, eps, lane);
#pragma unroll
    for (int j = 0; j < LN_MAX_V4; ++j)
        if (j < nv) {
            v[j].x *= c[j].x;
            v[j].y *= c[j].y;
            v[j].z *= c[j].z;
            v[j].w *= c[j].w;
        }
    ln_row<false>(v, nv, w, det_g, det_b, eps, lane, nullptr, out + row * w);
}

int owl_merge_ln(const float* x, int n, int N, int w, const float* post_g, const float* post_b, const float* det_g,
                 const float* det_b, float eps, __nv_bfloat16* out, cudaStream_t s) {
    if (n <= 0) return 0;
    check_ln_width(w);
    if (N < 2) fail(B200_ERR_INTERNAL, "owl_merge_ln: %d rows per image", N);
    const long long rows = (long long)n * (N - 1);
    owl_merge_ln_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(x, n, N, w, post_g, post_b, det_g, det_b, eps, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// One warp per patch row.  Each warp also forms the unit query u = t / |t| and |u| (E <= 1024 floats from L1): the
// text embedding reaches the head already normalised (OwlViTModel's text_embeds), and the head normalises it again
// with its 1e-6.  The two norms and the dot product are lane-strided sums, then a butterfly: a fixed order.
__global__ void __launch_bounds__(256) owl_class_logits_kernel(const float* __restrict__ c, int ldc, int M, int E,
                                                               const float* __restrict__ t, float* __restrict__ out) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    float tt = 0.f;
    for (int i = lane; i < E; i += 32) tt = fmaf(t[i], t[i], tt);
    const float tn = sqrtf(warp_sum(tt));
    const float* cr = c + row * ldc;
    float cc = 0.f, uu = 0.f, cu = 0.f;
    for (int i = lane; i < E; i += 32) {
        const float u = t[i] / tn, ci = cr[i];
        cc = fmaf(ci, ci, cc);
        uu = fmaf(u, u, uu);
        cu = fmaf(ci, u, cu);
    }
    cc = warp_sum(cc);
    uu = warp_sum(uu);
    cu = warp_sum(cu);
    if (lane == 0) {
        const float dot = cu / ((sqrtf(cc) + 1e-6f) * (sqrtf(uu) + 1e-6f));
        const float shift = cr[E], scale = cr[E + 1];
        const float elu = scale > 0.f ? scale : expm1f(scale);
        out[row] = (dot + shift) * (elu + 1.f);
    }
}

int owl_class_logits(const float* c, int ldc, int M, int E, const float* t, float* out, cudaStream_t s) {
    if (M <= 0) return 0;
    if (E <= 0 || ldc < E + 2) fail(B200_ERR_INTERNAL, "owl_class_logits: E %d, ldc %d", E, ldc);
    owl_class_logits_kernel<<<(M + 7) / 8, 256, 0, s>>>(c, ldc, M, E, t, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// One warp per patch row: the four dense2 dot products over the bf16 row (8 columns per lane per step), a butterfly
// each, then lanes 0..3 add the bias and the row's box bias and take the sigmoid.
__global__ void __launch_bounds__(256) owl_boxes_kernel(const __nv_bfloat16* __restrict__ a, int M, int w, int P,
                                                        const float* __restrict__ w2, const float* __restrict__ b2,
                                                        const float* __restrict__ box_bias, float* __restrict__ out) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    const __nv_bfloat16* ar = a + row * w;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int i4 = lane; i4 < w / 4; i4 += 32) {
        const float4 v = load4(ar, i4);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(w2 + (long long)j * w) + i4);
            acc[j] = fmaf(v.x, g.x, fmaf(v.y, g.y, fmaf(v.z, g.z, fmaf(v.w, g.w, acc[j]))));
        }
    }
    float r = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float sj = warp_sum(acc[j]);
        if (lane == j) r = sj;
    }
    if (lane < 4) {
        const float z = r + b2[lane] + box_bias[(row % P) * 4 + lane];
        out[row * 4 + lane] = 1.f / (1.f + expf(-z));
    }
}

int owl_boxes(const __nv_bfloat16* a, int M, int w, int P, const float* w2, const float* b2, const float* box_bias,
              float* out, cudaStream_t s) {
    if (M <= 0) return 0;
    if (w <= 0 || w % 4 != 0 || P <= 0) fail(B200_ERR_INTERNAL, "owl_boxes: width %d, %d patches", w, P);
    owl_boxes_kernel<<<(M + 7) / 8, 256, 0, s>>>(a, M, w, P, w2, b2, box_bias, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

void owl_box_bias(int G, float* out) {
    auto logit = [](double v) { return std::log(v + 1e-4) - std::log1p(-v + 1e-4); };
    const double size = logit(1.0 / G);
    for (int r = 0; r < G; ++r)
        for (int c = 0; c < G; ++c) {
            float* o = out + ((size_t)r * G + c) * 4;
            o[0] = (float)logit((double)(c + 1) / G);
            o[1] = (float)logit((double)(r + 1) / G);
            o[2] = (float)size;
            o[3] = (float)size;
        }
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

// Rows first .. first + count - 1 of the table for in_size -> out_size: a row depends on its index and the two sizes
// only, so the S rows a crop keeps are computed without the rest of the resized image's.
static ResampleTable precompute(int in_size, int out_size, int first, int count) {
    ResampleTable t;
    const double scale = (double)in_size / (double)out_size;
    double filterscale = scale;
    if (filterscale < 1.0) filterscale = 1.0;
    const double support = 2.0 * filterscale;
    t.ksize = (int)ceil(support) * 2 + 1;
    t.bounds.assign((size_t)count * 2, 0);
    t.coeffs.assign((size_t)count * t.ksize, 0);
    std::vector<double> k(t.ksize);
    for (int r = 0; r < count; ++r) {
        const int xx = first + r;
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
            t.coeffs[(size_t)r * t.ksize + x] =
                v < 0 ? (int)(-0.5 + v * (1 << PRECISION_BITS)) : (int)(0.5 + v * (1 << PRECISION_BITS));
        }
        t.bounds[(size_t)r * 2] = xmin;
        t.bounds[(size_t)r * 2 + 1] = xmax;
    }
    return t;
}

__device__ __forceinline__ uint8_t clip8(int v) {
    v >>= PRECISION_BITS;
    return (uint8_t)min(max(v, 0), 255);
}

// One image of a ragged resize.  Its tables hold the S rows of the window kept: bounds [S][2] = (first source pixel,
// taps) and coeffs [S][ksize], at int offsets into the packed table block.
struct ResizeDesc {
    const uint8_t* src;   // [h, w, 3]
    long long row0;       // its first row in the intermediate [sum_i h_i, S, 3]
    long long hb, hc;     // horizontal table: output column xo of the window
    long long vb, vc;     // vertical table: output row yo of the window
    int h, w, hk, vk;
};

// Image of intermediate row r: the last descriptor whose row0 <= r (row0 ascends, descriptor 0's is 0).
__device__ __forceinline__ int image_of_row(const ResizeDesc* __restrict__ d, int n, long long r) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (d[mid].row0 <= r) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// horizontal: every source row of every image -> tmp [rows, S, 3], the S output columns of its window
__global__ void resample_h_kernel(const ResizeDesc* __restrict__ d, int n, long long rows, int S,
                                  const int* __restrict__ tab, uint8_t* __restrict__ tmp) {
    // one search per block for the image of its first row; a block spans a few rows, so its threads step from there
    __shared__ int first;
    const long long i0 = (long long)blockIdx.x * blockDim.x;
    if (threadIdx.x == 0) first = image_of_row(d, n, i0 / S);
    __syncthreads();
    const long long i = i0 + threadIdx.x;
    if (i >= rows * S) return;
    const long long r = i / S;
    const int xo = (int)(i - r * S);
    int b = first;
    while (b + 1 < n && d[b + 1].row0 <= r) ++b;
    const ResizeDesc& D = d[b];
    const int xmin = tab[D.hb + 2 * xo], cnt = tab[D.hb + 2 * xo + 1];
    const int* k = tab + D.hc + (long long)xo * D.hk;
    const uint8_t* line = D.src + (r - D.row0) * D.w * 3;
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

// vertical: tmp [rows, S, 3] -> dst [n, S, S, 3], the S output rows of each image's window
__global__ void resample_v_kernel(const ResizeDesc* __restrict__ d, int n, int S, const int* __restrict__ tab,
                                  const uint8_t* __restrict__ tmp, uint8_t* __restrict__ dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long SS = (long long)S * S;
    if (i >= n * SS) return;
    const long long b = i / SS;
    const int p = (int)(i - b * SS);
    const int yo = p / S, xo = p - yo * S;
    const ResizeDesc& D = d[b];
    const int ymin = tab[D.vb + 2 * yo], cnt = tab[D.vb + 2 * yo + 1];
    const int* k = tab + D.vc + (long long)yo * D.vk;
    const uint8_t* col = tmp + ((D.row0 + ymin) * S + xo) * 3;
    int s0 = 1 << (PRECISION_BITS - 1), s1 = s0, s2 = s0;
    for (int y = 0; y < cnt; ++y) {
        const int c = k[y];
        const uint8_t* px = col + (long long)y * S * 3;
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

int resize_u8(const uint8_t* const* src, const int32_t* h, const int32_t* w, int n, int S, bool squash, uint8_t* dst,
              cudaStream_t s) {
    if (n <= 0) return 0;
    // descriptors, then the tables, in one block: one upload
    const size_t desc_bytes = (size_t)n * sizeof(ResizeDesc);
    static_assert(sizeof(ResizeDesc) % sizeof(int) == 0, "the tables follow the descriptors int-aligned");
    std::vector<ResizeDesc> desc((size_t)n);
    std::vector<int> tab;
    // (in, out, first) -> offsets of (bounds, coeffs) and ksize: one table per distinct resize of an axis in the call
    std::map<std::tuple<int, int, int>, std::tuple<long long, long long, int>> tables;
    auto table = [&](int in, int out, int first, long long& b, long long& c, int& k) {
        auto it = tables.find({in, out, first});
        if (it == tables.end()) {
            const ResampleTable t = precompute(in, out, first, S);
            const long long at = (long long)tab.size();
            tab.insert(tab.end(), t.bounds.begin(), t.bounds.end());
            tab.insert(tab.end(), t.coeffs.begin(), t.coeffs.end());
            it = tables.emplace(std::make_tuple(in, out, first), std::make_tuple(at, at + 2LL * S, t.ksize)).first;
        }
        std::tie(b, c, k) = it->second;
    };
    long long rows = 0;
    for (int i = 0; i < n; ++i) {
        int new_h = S, new_w = S, top = 0, left = 0;
        if (!squash) {
            // torchvision Resize(S): shortest side -> S, the other int(S * long / short); CenterCrop(S)
            if (w[i] <= h[i])
                new_h = (int)((double)((long long)S * h[i]) / (double)w[i]);   // int(S * long / short): true division
            else
                new_w = (int)((double)((long long)S * w[i]) / (double)h[i]);
            left = py_round_half_even((new_w - S) / 2.0);
            top = py_round_half_even((new_h - S) / 2.0);
        }
        // squash: PIL resize((S, S), BICUBIC) = torchvision Resize((S, S)) on a PIL image, nothing cropped.  An axis
        // that already has S pixels gets the identity coefficients (a single 1.0 tap), so running its pass is exact.
        ResizeDesc& D = desc[i];
        D.src = src[i];
        D.row0 = rows;
        D.h = h[i];
        D.w = w[i];
        table(w[i], new_w, left, D.hb, D.hc, D.hk);
        table(h[i], new_h, top, D.vb, D.vc, D.vk);
        rows += h[i];
    }
    std::vector<uint8_t> block(desc_bytes + tab.size() * sizeof(int));
    std::memcpy(block.data(), desc.data(), desc_bytes);
    std::memcpy(block.data() + desc_bytes, tab.data(), tab.size() * sizeof(int));
    {   // stream-ordered temporaries, released on `s` at the end of this block
        const DeviceBuffer<uint8_t> d_block(block.size(), s);
        MB_CUDA(cudaMemcpyAsync(d_block.get(), block.data(), block.size(), cudaMemcpyHostToDevice, s));
        // `block` is pageable and freed on return: the copy must be done before the kernels are even queued
        MB_CUDA(cudaStreamSynchronize(s));
        const ResizeDesc* d_desc = reinterpret_cast<const ResizeDesc*>(d_block.get());
        const int* d_tab = reinterpret_cast<const int*>(d_block.get() + desc_bytes);
        const DeviceBuffer<uint8_t> tmp((size_t)rows * S * 3, s);
        const long long nh = rows * S;
        resample_h_kernel<<<(unsigned)((nh + 255) / 256), 256, 0, s>>>(d_desc, n, rows, S, d_tab, tmp.get());
        MB_CUDA(cudaGetLastError());
        const long long nv = (long long)n * S * S;
        resample_v_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, s>>>(d_desc, n, S, d_tab, tmp.get(), dst);
        MB_CUDA(cudaGetLastError());
    }
    return 2;
}

// the uniform batch [n, h, w, 3]: every image's pointer into it, one size
static int resize_uniform_u8(const uint8_t* src, int n, int h, int w, int S, bool squash, uint8_t* dst,
                             cudaStream_t s) {
    if (n <= 0) return 0;
    std::vector<const uint8_t*> ptr((size_t)n);
    for (int i = 0; i < n; ++i) ptr[i] = src + (size_t)i * h * w * 3;
    const std::vector<int32_t> hs((size_t)n, h), ws((size_t)n, w);
    return resize_u8(ptr.data(), hs.data(), ws.data(), n, S, squash, dst, s);
}

int resize_crop_u8(const uint8_t* src, int n, int h, int w, int S, uint8_t* dst, cudaStream_t s) {
    return resize_uniform_u8(src, n, h, w, S, false, dst, s);
}

int resize_squash_u8(const uint8_t* src, int n, int h, int w, int S, uint8_t* dst, cudaStream_t s) {
    return resize_uniform_u8(src, n, h, w, S, true, dst, s);
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

// HD: the head dim, 64 or 96 (CoCa ViT-L-14's attentional pooler: 8 heads over 768 columns).  At HD 96 pass 3 gives
// lane l columns 2l, 2l + 1 and, for l < 16, 64 + 2l, 65 + 2l.
template <int HD>
__global__ void __launch_bounds__(MAP_THREADS) map_attention_kernel(const float* __restrict__ q, long long q_stride,
                                                                    const __nv_bfloat16* __restrict__ kv, int S, int W,
                                                                    __nv_bfloat16* __restrict__ out) {
    // 1 / sqrt(HD) * log2(e)
    constexpr float SCALE = (HD == 64 ? 0.125f : 0.10206207261596575f) * 1.4426950408889634f;
    extern __shared__ float logit[];   // [S]
    __shared__ float qs[HD];
    __shared__ float red[4];
    __shared__ float part[4][HD];
    const int b = blockIdx.x, h = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid < HD) qs[tid] = q[b * q_stride + h * HD + tid] * SCALE;
    __syncthreads();
    const long long ld = 2LL * W;
    const __nv_bfloat16* keys = kv + (long long)b * S * ld + h * HD;
    const __nv_bfloat16* vals = keys + W;
    float mx = -INFINITY;
    for (int s = tid; s < S; s += MAP_THREADS) {
        const uint4* k4 = reinterpret_cast<const uint4*>(keys + s * ld);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < HD / 8; ++j) {
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
    if constexpr (HD == 64) {
        float2 acc = make_float2(0.f, 0.f);
        for (int s = warp; s < S; s += 4) {
            const float p = logit[s];
            const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(vals + s * ld + 2 * lane));
            acc.x = fmaf(p, f.x, acc.x);
            acc.y = fmaf(p, f.y, acc.y);
        }
        part[warp][2 * lane] = acc.x;
        part[warp][2 * lane + 1] = acc.y;
    } else {
        const bool hi = lane < 16;   // lanes 0..15 also own columns 64 + 2l, 65 + 2l
        float2 acc = make_float2(0.f, 0.f), acc2 = make_float2(0.f, 0.f);
        for (int s = warp; s < S; s += 4) {
            const float p = logit[s];
            const __nv_bfloat162* v2 = reinterpret_cast<const __nv_bfloat162*>(vals + s * ld);
            const float2 f = __bfloat1622float2(v2[lane]);
            acc.x = fmaf(p, f.x, acc.x);
            acc.y = fmaf(p, f.y, acc.y);
            if (hi) {
                const float2 g = __bfloat1622float2(v2[32 + lane]);
                acc2.x = fmaf(p, g.x, acc2.x);
                acc2.y = fmaf(p, g.y, acc2.y);
            }
        }
        part[warp][2 * lane] = acc.x;
        part[warp][2 * lane + 1] = acc.y;
        if (hi) {
            part[warp][64 + 2 * lane] = acc2.x;
            part[warp][65 + 2 * lane] = acc2.y;
        }
    }
    __syncthreads();
    if (tid < HD) {
        const float o = ((part[0][tid] + part[1][tid]) + part[2][tid]) + part[3][tid];
        out[(long long)b * W + h * HD + tid] = __float2bfloat16_rn(o / sum);
    }
}

int map_attention(const float* q, long long q_stride, const __nv_bfloat16* kv, int n, int S, int W, int heads,
                  __nv_bfloat16* out, cudaStream_t s) {
    if (n <= 0) return 0;
    if (heads <= 0 || (W != heads * 64 && W != heads * 96))
        fail(B200_ERR_UNSUPPORTED, "map_attention: head_dim must be 64 or 96 (width %d, heads %d)", W, heads);
    if (S <= 0 || S > MAP_MAX_TOKENS) fail(B200_ERR_UNSUPPORTED, "map_attention: %d tokens (1..%d)", S, MAP_MAX_TOKENS);
    const dim3 grid((unsigned)n, (unsigned)heads);
    if (W == heads * 64)
        map_attention_kernel<64><<<grid, MAP_THREADS, (size_t)S * sizeof(float), s>>>(q, q_stride, kv, S, W, out);
    else
        map_attention_kernel<96><<<grid, MAP_THREADS, (size_t)S * sizeof(float), s>>>(q, q_stride, kv, S, W, out);
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

// ------------------------------------------------------------------------------------------------ LanguageBind video
// LanguageBind's heads (languagebind/__init__.py:55-64, video/modeling_video.py:766-771):
//   (1) frame_mean_ln_kernel  one warp per item: LayerNorm of each of its T pooled rows, then their mean -> pooled
//   (2) head_proj_kernel      the CLIP head's projection
//   (3) head_scale_kernel     one warp per item: v / |v| * scale, then, if normalize, / its norm again (no epsilons)
__global__ void __launch_bounds__(256) frame_mean_ln_kernel(const float* __restrict__ x, int N, int T,
                                                            const int32_t* __restrict__ row_in_seq,
                                                            const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float eps, int n, int w,
                                                            float* __restrict__ pooled) {
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= n) return;
    const int r = row_in_seq ? row_in_seq[b] : 0;
    float* dst = pooled + (long long)b * w;
    for (int t = 0; t < T; ++t) {
        const float* src = x + (((long long)b * T + t) * N + r) * w;
        float s = 0.f;
        for (int i = lane; i < w; i += 32) s += src[i];
        const float mean = warp_sum(s) / (float)w;
        float q = 0.f;
        for (int i = lane; i < w; i += 32) {
            const float d = src[i] - mean;
            q += d * d;
        }
        const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)w + eps);
        // each lane owns the same columns for every t: the sum needs no synchronisation
        for (int i = lane; i < w; i += 32) {
            const float y = (src[i] - mean) * rstd * gamma[i] + beta[i];
            dst[i] = t == 0 ? y : dst[i] + y;
        }
    }
    for (int i = lane; i < w; i += 32) dst[i] = dst[i] / (float)T;
}

__global__ void __launch_bounds__(256) head_scale_kernel(float* __restrict__ out, int n, int E, float scale,
                                                         int normalize) {
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= n) return;
    float* row = out + (long long)b * E;
    float ss = 0.f;
    for (int i = lane; i < E; i += 32) ss += row[i] * row[i];
    const float nrm = sqrtf(warp_sum(ss));
    ss = 0.f;
    for (int i = lane; i < E; i += 32) {
        const float v = row[i] / nrm * scale;
        row[i] = v;
        ss += v * v;
    }
    if (!normalize) return;
    const float nrm2 = sqrtf(warp_sum(ss));
    for (int i = lane; i < E; i += 32) row[i] = row[i] / nrm2;
}

int frame_mean_head(const float* x, int N, int T, const int32_t* row_in_seq, const float* gamma, const float* beta,
                    float eps, const float* proj, int n, int w, int E, float scale, int normalize, float* out,
                    float* pooled_ws, cudaStream_t s) {
    if (n <= 0) return 0;
    if (w % 4 != 0 || (size_t)HEAD_IMGS * w * sizeof(float) > 40 * 1024)
        fail(B200_ERR_UNSUPPORTED, "frame_mean_head: width %d unsupported", w);
    if (T < 1) fail(B200_ERR_INVALID_ARG, "frame_mean_head: T %d must be positive", T);
    frame_mean_ln_kernel<<<(n + 7) / 8, 256, 0, s>>>(x, N, T, row_in_seq, gamma, beta, eps, n, w, pooled_ws);
    MB_CUDA(cudaGetLastError());
    const dim3 grid((n + HEAD_IMGS - 1) / HEAD_IMGS, (E + HEAD_COLS - 1) / HEAD_COLS);
    head_proj_kernel<<<grid, 256, (size_t)HEAD_IMGS * w * sizeof(float), s>>>(pooled_ws, proj, nullptr, n, w, E, out);
    MB_CUDA(cudaGetLastError());
    head_scale_kernel<<<(n + 7) / 8, 256, 0, s>>>(out, n, E, scale, normalize);
    MB_CUDA(cudaGetLastError());
    return 3;
}

// x[r] += temb[(r / N) % T] (when temb != NULL), then h[r] = bf16(LN(x[r])): one warp per row, the row read once.
__global__ void __launch_bounds__(256) temporal_embed_ln_kernel(float* __restrict__ x, const float* __restrict__ temb,
                                                                int N, int T, const float* __restrict__ gamma,
                                                                const float* __restrict__ beta, float eps, int rows,
                                                                int w, __nv_bfloat16* __restrict__ h) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int nv = w / 128;
    float* src = x + (long long)row * w;
    float4 v[LN_MAX_V4];
#pragma unroll
    for (int j = 0; j < LN_MAX_V4; ++j)
        if (j < nv) v[j] = load4(src, lane + 32 * j);
    if (temb) {
        const float* e = temb + (long long)((row / N) % T) * w;
#pragma unroll
        for (int j = 0; j < LN_MAX_V4; ++j)
            if (j < nv) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(e) + lane + 32 * j);
                v[j] = make_float4(v[j].x + a.x, v[j].y + a.y, v[j].z + a.z, v[j].w + a.w);
                reinterpret_cast<float4*>(src)[lane + 32 * j] = v[j];
            }
    }
    ln_row<false, LN_MAX_V4>(v, nv, w, gamma, beta, eps, lane, nullptr, h + (long long)row * w);
}

int temporal_embed_ln(float* x, const float* temb, int N, int T, const float* gamma, const float* beta, float eps,
                      int rows, int w, __nv_bfloat16* h, cudaStream_t s) {
    if (rows <= 0) return 0;
    check_ln_width(w);
    if (N <= 0 || T <= 0) fail(B200_ERR_INVALID_ARG, "temporal_embed_ln: N %d and T %d must be positive", N, T);
    temporal_embed_ln_kernel<<<(rows + 7) / 8, 256, 0, s>>>(x, temb, N, T, gamma, beta, eps, rows, w, h);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// Eight lanes per (item, token, head): lane l owns columns 8 l .. 8 l + 7 of the head, read as 16-byte loads.  For
// each query frame i the group reads q_i and the T frames' k and v rows (k and v again for every query, from L1 / L2:
// held in registers across the queries they would take 128 of them at T = 8), sums each score over its 8 lanes by
// shuffles, and takes the softmax in fp32 (exp2 of logits pre-scaled by log2(e) / sqrt(64)), the weighted sum of v and
// one 16-byte bf16 store.  Frame t of an (item, token) pair is row (b T + t) N + token of the packed buffers: no
// (b n) t copy.  A group past the end reads the last group's rows (every lane of a warp takes part in the shuffles) and
// stores nothing.
__device__ __forceinline__ void unpack8(const uint4 u, float (&f)[8]) {
    const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        f[2 * i] = __uint_as_float(w4[i] << 16);
        f[2 * i + 1] = __uint_as_float(w4[i] & 0xffff0000u);
    }
}

template <int TMAX>
__global__ void __launch_bounds__(256) temporal_attention_kernel(const __nv_bfloat16* __restrict__ qkv, int N, int T,
                                                                 int H, long long groups, float scale_log2,
                                                                 __nv_bfloat16* __restrict__ out) {
    const long long g0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const bool valid = g0 < groups;
    const long long g = valid ? g0 : groups - 1;
    const int l = threadIdx.x & 7;
    const int h = (int)(g % H);
    const long long bn = g / H;
    const int tok = (int)(bn % N);
    const long long b = bn / N;
    const int W = H * 64;
    const long long ld = 3LL * W, step = (long long)N * ld;   // frame t's row: row0 + t N
    const long long row0 = b * T * N + tok;
    const __nv_bfloat16* base = qkv + row0 * ld + h * 64 + l * 8;
    for (int i = 0; i < T; ++i) {
        float q[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(base + i * step)), q);
        float s[TMAX];
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < TMAX; ++j)
            if (j < T) {
                float kf[8];
                unpack8(__ldg(reinterpret_cast<const uint4*>(base + j * step + W)), kf);
                float d = 0.f;
#pragma unroll
                for (int c = 0; c < 8; ++c) d = fmaf(q[c], kf[c], d);
                d += __shfl_xor_sync(0xffffffffu, d, 1);
                d += __shfl_xor_sync(0xffffffffu, d, 2);
                d += __shfl_xor_sync(0xffffffffu, d, 4);
                s[j] = d * scale_log2;
                m = fmaxf(m, s[j]);
            }
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < TMAX; ++j)
            if (j < T) {
                const float p = exp2f(s[j] - m);
                sum += p;
                float vf[8];
                unpack8(__ldg(reinterpret_cast<const uint4*>(base + j * step + 2 * W)), vf);
#pragma unroll
                for (int c = 0; c < 8; ++c) acc[c] = fmaf(p, vf[c], acc[c]);
            }
        if (valid) {
            const float inv = 1.0f / sum;
            uint4 o;
            o.x = pack_bf16x2(acc[0] * inv, acc[1] * inv);
            o.y = pack_bf16x2(acc[2] * inv, acc[3] * inv);
            o.z = pack_bf16x2(acc[4] * inv, acc[5] * inv);
            o.w = pack_bf16x2(acc[6] * inv, acc[7] * inv);
            *reinterpret_cast<uint4*>(out + (row0 + (long long)i * N) * W + h * 64 + l * 8) = o;
        }
    }
}

int temporal_attention(const __nv_bfloat16* qkv, int n, int T, int N, int W, int heads, __nv_bfloat16* out,
                       cudaStream_t s) {
    if (n <= 0) return 0;
    if (T < 1 || T > TEMPORAL_MAX_FRAMES)
        fail(B200_ERR_INVALID_ARG, "temporal_attention: T %d must be 1..%d", T, TEMPORAL_MAX_FRAMES);
    if (heads <= 0 || W != heads * 64 || N <= 0)
        fail(B200_ERR_UNSUPPORTED, "temporal_attention: heads of 64 only (W %d, heads %d, N %d)", W, heads, N);
    const long long groups = (long long)n * N * heads;
    const unsigned blocks = (unsigned)((groups * 8 + 255) / 256);
    const float scale_log2 = 0.125f * 1.4426950408889634f;
    if (T <= 8)
        temporal_attention_kernel<8><<<blocks, 256, 0, s>>>(qkv, N, T, heads, groups, scale_log2, out);
    else
        temporal_attention_kernel<TEMPORAL_MAX_FRAMES>
            <<<blocks, 256, 0, s>>>(qkv, N, T, heads, groups, scale_log2, out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

// One thread per output pixel (f, y, x) of the S x S crop, all three channels: the source point in the frame of the
// resized pixel (y + top, x + left) by F.interpolate's rule (align_corners False: (dst + 0.5) h / nh - 0.5 as one fma,
// clamped at 0; the far tap clamped to the last row / column), bilinear over the uint8 values in fp32, then / 255 and Normalize.
// The reference normalises before it resizes; the bilinear weights sum to 1, so the two orders differ by rounding.
__global__ void __launch_bounds__(256) video_resize_crop_kernel(const uint8_t* __restrict__ src, long long total, int H,
                                                                int W, int S, int top, int left, float sy, float sx,
                                                                float3 mean, float3 stdv, float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const long long plane = (long long)S * S;
    const long long f = i / plane;
    const int p = (int)(i - f * plane), y = p / S, x = p - y * S;
    const float fy = fmaxf(fmaf(sy, (float)(y + top) + 0.5f, -0.5f), 0.f);
    const float fx = fmaxf(fmaf(sx, (float)(x + left) + 0.5f, -0.5f), 0.f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const uint8_t* img = src + f * H * W * 3;
    const uint8_t *a = img + ((long long)y0 * W + x0) * 3, *b = img + ((long long)y0 * W + x1) * 3;
    const uint8_t *c = img + ((long long)y1 * W + x0) * 3, *d = img + ((long long)y1 * W + x1) * 3;
    const float m[3] = {mean.x, mean.y, mean.z}, sd[3] = {stdv.x, stdv.y, stdv.z};
    float* o = out + f * 3 * plane + p;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float v = hy * (hx * (float)a[ch] + lx * (float)b[ch]) + ly * (hx * (float)c[ch] + lx * (float)d[ch]);
        o[ch * plane] = (v / 255.f - m[ch]) / sd[ch];
    }
}

void video_resize_geometry(int h, int w, int S, int* nh, int* nw, int* top, int* left) {
    // pytorchvideo's short_side_scale: the short side to S, the long one to floor(long / short * S) in double
    if (w < h) {
        *nh = (int)std::floor((double)h / w * S);
        *nw = S;
    } else {
        *nh = S;
        *nw = (int)std::floor((double)w / h * S);
    }
    // torchvision's CenterCropVideo: int(round((size - S) / 2.0)), Python's round (half to even)
    *top = py_round_half_even((*nh - S) / 2.0);
    *left = py_round_half_even((*nw - S) / 2.0);
}

int video_resize_crop(const uint8_t* src, long long frames, int h, int w, int S, const float* mean, const float* std_,
                      float* out, cudaStream_t s) {
    if (frames <= 0) return 0;
    if (h <= 0 || w <= 0 || S <= 0) fail(B200_ERR_INVALID_ARG, "video_resize_crop: bad size %d x %d -> %d", h, w, S);
    int nh, nw, top, left;
    video_resize_geometry(h, w, S, &nh, &nw, &top, &left);
    const long long total = frames * S * S;
    video_resize_crop_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
        src, total, h, w, S, top, left, (float)h / (float)nh, (float)w / (float)nw,
        make_float3(mean[0], mean[1], mean[2]), make_float3(std_[0], std_[1], std_[2]), out);
    MB_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace kernels
}  // namespace mb
