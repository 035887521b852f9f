// Diagnostic entry points: run one encoder kernel on the caller's device buffers (kernel-level numerics tests).
#include <algorithm>
#include <vector>

#include "attention.cuh"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.cuh"
#include "score.cuh"

using namespace mb;

namespace {

using bf16 = __nv_bfloat16;

struct Scratch {   // a stream and the device buffers of one timing call
    UniqueStream stream = make_stream(cudaStreamDefault);
    cudaStream_t s = stream.get();
    std::vector<DeviceBuffer<uint8_t>> bufs;
    template <class T>
    T* alloc(size_t n) {
        bufs.emplace_back(std::max<size_t>(n * sizeof(T), 16));
        return reinterpret_cast<T*>(bufs.back().get());
    }
};

// pseudo-random values in [-1, 1) (kernel timing probes: no 200 MB host upload)
__device__ __forceinline__ float fill_value(long long i, uint32_t seed) {
    uint32_t x = (uint32_t)i * 2654435761u + seed;
    x ^= x >> 16;
    x *= 0x85ebca6bu;
    x ^= x >> 13;
    return (float)(x & 0xFFFF) / 32768.0f - 1.0f;
}
__global__ void fill_bf16_kernel(__nv_bfloat16* dst, long long n, uint32_t seed) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = __float2bfloat16_rn(fill_value(i, seed));
}
__global__ void fill_f32_kernel(float* dst, long long n, uint32_t seed) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = fill_value(i, seed);
}

void require_device(int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        fail(B200_ERR_NO_DEVICE, "CUDA device %d not available (marqo_b200 has no CPU fallback)", device);
    }
}

}  // namespace

extern "C" {

int b200_debug_patch_embed(int device, const uint8_t* hwc, int n, int S, int patch, const float* conv_w, int N,
                           const float* mean3, const float* std3, const float* cls, const float* pos,
                           const float* bias, float* out, int ldo, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(hwc && conv_w && mean3 && std3 && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && patch > 0 && S % patch == 0 && N > 0 && N % 32 == 0, "bad shape");
        const bool vit = pos != nullptr;
        if (vit)
            MB_CHECK_ARG(bias == nullptr && ldo == N, "the ViT form has no bias and compact rows (ldo %d, N %d)", ldo, N);
        else
            MB_CHECK_ARG(cls == nullptr && ldo >= N && ldo % 8 == 0,
                         "the stem form has no class row, and ldo %d must be a multiple of 8, >= N %d", ldo, N);
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        const int G = (S / patch) * (S / patch);
        DeviceBuffer<bf16> wg((size_t)N * gemm::patch_gather_k(patch));
        kernels::patch_weight_rows(conv_w, N, patch, gemm::patch_gather_kbpd(patch), wg.get(), s);
        gemm::Epilogue ep;
        ep.out = out;
        ep.ldo = ldo;
        ep.out_fp32 = 1;
        if (vit) {
            // as forward_vit does: x = pos (+ cls), then the gather GEMM adds conv1 onto it in place
            kernels::vit_embed_rows(out, cls, pos, n, G + (cls != nullptr), N, s);
            ep.residual = out;
            ep.ldr = N;
        } else {
            ep.bias = bias;   // as forward_convnext's stem: conv + bias, no residual
        }
        gemm::PatchGather pg;
        pg.img = hwc;
        pg.n = n;
        pg.S = S;
        pg.patch = patch;
        pg.cls = cls != nullptr;
        for (int i = 0; i < 3; ++i) {
            pg.mean[i] = mean3[i];
            pg.std[i] = std3[i];
        }
        gemm::launch_patch_embed(pg, wg.get(), N, ep, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_gemm(int device, const void* A, int lda, const void* W, const float* bias, const float* residual, int ldr,
                    void* out, int ldo, int out_bf16, int act, int M, int N, int K, int sms, int* kernel_out,
                    void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(A && W && out, "NULL buffer");
        MB_CHECK_ARG(M > 0 && N > 0 && K > 0 && lda >= K && ldo >= N && (!residual || ldr >= N) && sms >= 0, "bad shape");
        MB_CHECK_ARG(!(residual == out && out_bf16), "the in-place residual is fp32");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        gemm::Epilogue ep;
        ep.bias = bias;
        ep.residual = residual;
        ep.ldr = ldr;
        ep.act = act;
        ep.out = out;
        ep.ldo = ldo;
        ep.out_fp32 = out_bf16 ? 0 : 1;
        const int kernel = gemm::launch(static_cast<const bf16*>(A), lda, static_cast<const bf16*>(W), M, N, K, ep,
                                        sms > 0 ? sms : sm_count(device), s);
        if (kernel_out) *kernel_out = kernel;
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_index_scan_kernel(b200_index* ix, int force_streamed, int* last_kernel) {
    return guarded([&] { score::debug_scan_kernel(ix, force_streamed, last_kernel); });
}

int b200_debug_index_last_scan(b200_index* ix, int* nq, int* grid, float* eps, float* queries, float* list_score,
                               int32_t* list_row, int32_t* list_doc) {
    return guarded([&] { score::debug_last_scan(ix, nq, grid, eps, queries, list_score, list_row, list_doc); });
}

int b200_debug_gemm_time(int device, int M, int N, int K, int act, int out_bf16, int has_bias, int residual_in_place,
                         int iters, float* out_ms) {
    return guarded([&] {
        MB_CHECK_ARG(out_ms != nullptr, "NULL buffer");
        MB_CHECK_ARG(M > 0 && N > 0 && K > 0 && iters > 0, "M, N, K, iters must be positive");
        MB_CHECK_ARG(!(residual_in_place && out_bf16), "the in-place residual is fp32");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        __nv_bfloat16* dA = sc.alloc<__nv_bfloat16>((size_t)M * K);
        __nv_bfloat16* dW = sc.alloc<__nv_bfloat16>((size_t)N * K);
        const long long na = (long long)M * K, nw = (long long)N * K, no = (long long)M * N;
        fill_bf16_kernel<<<(unsigned)((na + 255) / 256), 256, 0, sc.s>>>(dA, na, 12345u);
        fill_bf16_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, sc.s>>>(dW, nw, 777u);
        gemm::Epilogue ep;
        ep.act = act;
        ep.ldo = N;
        if (has_bias) {
            float* dBias = sc.alloc<float>((size_t)N);
            fill_f32_kernel<<<(unsigned)((N + 255) / 256), 256, 0, sc.s>>>(dBias, N, 99u);
            ep.bias = dBias;
        }
        if (out_bf16) {
            ep.out = sc.alloc<__nv_bfloat16>((size_t)no);
        } else {
            float* dOut = sc.alloc<float>((size_t)no);
            fill_f32_kernel<<<(unsigned)((no + 255) / 256), 256, 0, sc.s>>>(dOut, no, 4242u);
            ep.out = dOut;
            ep.out_fp32 = 1;
            if (residual_in_place) {   // residual == out, as run_layers updates x
                ep.residual = dOut;
                ep.ldr = N;
            }
        }
        MB_CUDA(cudaGetLastError());
        const int sms = sm_count(device);
        UniqueEvent e0 = make_event(), e1 = make_event();
        for (int i = 0; i < 3; ++i) gemm::launch(dA, K, dW, M, N, K, ep, sms, sc.s);   // warm-up
        MB_CUDA(cudaEventRecord(e0.get(), sc.s));
        for (int i = 0; i < iters; ++i) gemm::launch(dA, K, dW, M, N, K, ep, sms, sc.s);
        MB_CUDA(cudaEventRecord(e1.get(), sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
        float ms = 0.f;
        MB_CUDA(cudaEventElapsedTime(&ms, e0.get(), e1.get()));
        *out_ms = ms / (float)iters;
    });
}

int b200_debug_attention(int device, const void* qkv, int B, int S, int W, int H, int mask, const int32_t* kv_len,
                         const float* rel_bias, int smax, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(qkv && out, "NULL buffer");
        MB_CHECK_ARG(B > 0 && S > 0 && W > 0 && H > 0, "B, S, W, H must be positive");
        MB_CHECK_ARG(!rel_bias || smax > 0, "smax must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        attention::RelBias bias;
        DeviceBuffer<float> table;
        std::vector<float> scaled;
        if (rel_bias) {   // the kernels add it in the log2 domain
            scaled.assign(rel_bias, rel_bias + (size_t)H * (2 * smax - 1));
            for (float& v : scaled) v *= 1.4426950408889634f;
            table = DeviceBuffer<float>(scaled.size());
            MB_CUDA(cudaMemcpyAsync(table.get(), scaled.data(), scaled.size() * 4, cudaMemcpyHostToDevice, s));
            bias.table = table.get();
            bias.smax = smax;
        }
        attention::launch(static_cast<const bf16*>(qkv), static_cast<bf16*>(out), B, S, W, H, mask, kv_len, bias, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_attention_padded(int device, const void* qkv, int B, int S, int W, int H, int model_hd, int mask,
                                const int32_t* kv_len, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(qkv && out, "NULL buffer");
        MB_CHECK_ARG(B > 0 && S > 0 && W > 0 && H > 0 && model_hd > 0, "B, S, W, H, model_hd must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        attention::launch(static_cast<const bf16*>(qkv), static_cast<bf16*>(out), B, S, W, H, mask, kv_len,
                          attention::RelBias{}, s, model_hd);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_attention_time(int device, int B, int S, int W, int H, int mask, int rel_bias, int iters, float* out_ms) {
    return guarded([&] {
        MB_CHECK_ARG(out_ms != nullptr, "NULL buffer");
        MB_CHECK_ARG(B > 0 && S > 0 && W > 0 && H > 0 && iters > 0, "B, S, W, H, iters must be positive");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const size_t M = (size_t)B * S;
        __nv_bfloat16* dq = sc.alloc<__nv_bfloat16>(M * 3 * W);
        __nv_bfloat16* dO = sc.alloc<__nv_bfloat16>(M * W);
        const long long n = (long long)(M * 3 * W);
        fill_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, sc.s>>>(dq, n, 12345u);
        attention::RelBias bias;
        if (rel_bias) {
            const long long nb = (long long)H * (2 * S - 1);
            float* table = sc.alloc<float>((size_t)nb);
            fill_f32_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, sc.s>>>(table, nb, 99u);
            bias.table = table;
            bias.smax = S;
        }
        MB_CUDA(cudaGetLastError());
        int32_t* dlen = nullptr;
        if (mask == attention::MASK_KEYLEN) {
            const std::vector<int32_t> lens((size_t)B, S);
            dlen = sc.alloc<int32_t>(lens.size());
            MB_CUDA(cudaMemcpy(dlen, lens.data(), lens.size() * 4, cudaMemcpyHostToDevice));
        }
        UniqueEvent e0 = make_event(), e1 = make_event();
        for (int i = 0; i < 3; ++i) attention::launch(dq, dO, B, S, W, H, mask, dlen, bias, sc.s);   // warm-up
        MB_CUDA(cudaEventRecord(e0.get(), sc.s));
        for (int i = 0; i < iters; ++i) attention::launch(dq, dO, B, S, W, H, mask, dlen, bias, sc.s);
        MB_CUDA(cudaEventRecord(e1.get(), sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
        float ms = 0.f;
        MB_CUDA(cudaEventElapsedTime(&ms, e0.get(), e1.get()));
        *out_ms = ms / (float)iters;
    });
}

int b200_debug_layernorm(int device, const float* x, long long in_stride, const float* gamma, const float* beta, float eps,
                         int rows, int w, float* out_f32, void* out_bf16, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && gamma && beta && (out_f32 || out_bf16), "NULL buffer");
        MB_CHECK_ARG(rows > 0 && w > 0 && in_stride >= 0, "rows, w must be positive");
        if (in_stride == 0) in_stride = w;
        MB_CHECK_ARG(in_stride >= w, "in_stride %lld < w %d", in_stride, w);
        MB_CHECK_ARG(out_f32 != x || in_stride == w, "in place needs compact rows");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::layernorm(x, in_stride, gamma, beta, eps, rows, w, out_f32, static_cast<bf16*>(out_bf16), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_layernorm_bf16(int device, const void* x, long long in_stride, const float* gamma, const float* beta,
                              float eps, int rows, int w, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && gamma && beta && out, "NULL buffer");
        MB_CHECK_ARG(rows > 0 && w > 0 && in_stride >= 0, "rows, w must be positive");
        if (in_stride == 0) in_stride = w;
        MB_CHECK_ARG(in_stride >= w, "in_stride %lld < w %d", in_stride, w);
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::layernorm_bf16(static_cast<const bf16*>(x), in_stride, gamma, beta, eps, rows, w, static_cast<bf16*>(out),
                                s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_rope_qk(int device, void* qkv, int n, int G, int w, int ref, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(qkv != nullptr, "NULL buffer");
        MB_CHECK_ARG(n > 0 && G > 0 && ref > 0 && w > 0 && w % 64 == 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        std::vector<float> table((size_t)G * G * 64);
        kernels::rope_table(G, ref, table.data());
        DeviceBuffer<float> dt(table.size());
        MB_CUDA(cudaMemcpyAsync(dt.get(), table.data(), table.size() * sizeof(float), cudaMemcpyHostToDevice, s));
        kernels::rope_qk(static_cast<bf16*>(qkv), n, G * G + 1, 1, w, dt.get(), kernels::RopePairing::INTERLEAVED, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_rope_qk_half(int device, void* qkv, int n, int S, int w, float theta, float ntk_factor, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(qkv != nullptr, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && w % 64 == 0, "bad shape");
        MB_CHECK_ARG(theta > 0.f && ntk_factor >= 1.f, "rope_theta must be positive and rope_ntk_factor >= 1");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        std::vector<float> table((size_t)S * 64);
        kernels::rope_table_ntk(S, theta, ntk_factor, table.data());
        DeviceBuffer<float> dt(table.size());
        MB_CUDA(cudaMemcpyAsync(dt.get(), table.data(), table.size() * sizeof(float), cudaMemcpyHostToDevice, s));
        kernels::rope_qk(static_cast<bf16*>(qkv), n, S, 0, w, dt.get(), kernels::RopePairing::HALF, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_geglu(int device, const void* in, int rows, int h, void* out, long long ldo, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(in && out, "NULL buffer");
        MB_CHECK_ARG(rows > 0 && h > 0 && h % 8 == 0, "rows must be positive and h a positive multiple of 8");
        MB_CHECK_ARG(ldo >= h && ldo % 8 == 0, "ldo %lld must be a multiple of 8, >= %d", ldo, h);
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::geglu(static_cast<const bf16*>(in), rows, h, static_cast<bf16*>(out), ldo, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_swiglu_ln(int device, const void* in, int rows, int h, const float* gamma, const float* beta, float eps,
                         void* out, long long ldo, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(in && gamma && beta && out, "NULL buffer");
        MB_CHECK_ARG(rows > 0 && h > 0, "rows, h must be positive");
        const int hp = (int)round_up((size_t)h, 64);
        MB_CHECK_ARG(ldo >= hp && ldo % 8 == 0, "ldo %lld must be a multiple of 8, >= %d", ldo, hp);
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::swiglu_ln(static_cast<const bf16*>(in), rows, hp, h, gamma, beta, eps, static_cast<bf16*>(out), ldo, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_clip_text_embed(int device, const int32_t* ids, const float* tok, const float* pos, int n, int S, int w,
                               int vocab, float* x, int32_t* eot, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(ids && tok && pos && x && eot, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && w % 4 == 0 && vocab > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::clip_text_embed(ids, tok, pos, n, S, w, vocab, x, eot, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_clip_text_embed_cls(int device, const int32_t* ids, const float* tok, const float* pos, const float* cls,
                                   int n, int S, int w, int vocab, float* x, int32_t* eot, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(ids && tok && pos && cls && x && eot, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 1 && w > 0 && w % 4 == 0 && vocab > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::clip_text_embed(ids, tok, pos, n, S, w, vocab, x, eot, s, cls);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_embed_ln(int device, const int32_t* ids, const int32_t* mask, const float* word, const float* pos,
                        int pos_rows, const float* type0, const float* gamma, const float* beta, float eps, int n, int S,
                        int w, int vocab, int pad, float* x, void* h, int32_t* kv_len, const int32_t* type_ids,
                        int type_rows, void* stream) {
    return guarded([&] {
        const bool roberta = pad >= 0;
        MB_CHECK_ARG(!type_ids || (!roberta && pos && type_rows > 0), "token-type ids: BERT with positions and rows");
        // pos NULL: the BERT embedding without a position row (GTE)
        MB_CHECK_ARG(ids && word && (pos || !roberta) && gamma && beta && x && h && kv_len, "NULL buffer");
        MB_CHECK_ARG(roberta || type0, "the BERT embedding always adds token-type row 0");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && vocab > 0, "bad shape");
        MB_CHECK_ARG(!pos || pos_rows >= (roberta ? pad + S + 1 : S), "%d position rows are too few", pos_rows);
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        if (roberta)
            kernels::roberta_embed_ln(ids, mask, word, pos, type0, gamma, beta, eps, n, S, w, vocab, pad, x,
                                      static_cast<bf16*>(h), kv_len, s);
        else
            kernels::bert_embed_ln(ids, mask, word, pos, type0, gamma, beta, eps, n, S, w, vocab, x, static_cast<bf16*>(h),
                                   kv_len, s, type_ids, type_ids ? type_rows : 1);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_clip_head(int device, const float* x, int S, const int32_t* row_in_seq, const float* gamma,
                         const float* beta, float eps, const float* proj, int n, int w, int E, int normalize, float* out,
                         void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && gamma && beta && proj && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && E > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        DeviceBuffer<float> pooled((size_t)n * w);
        kernels::clip_head(x, S, row_in_seq, gamma, beta, eps, proj, n, w, E, normalize, out, pooled.get(), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_bert_head(int device, const float* x, const int32_t* kv_len, int n, int S, int w, int pool, int normalize,
                         float* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && kv_len && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && (pool == 0 || pool == 1), "bad shape or pool");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::bert_head(x, kv_len, n, S, w, pool, normalize, out, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_text_head(int device, const float* x, const int32_t* kv_len, int n, int S, int w, const float* proj,
                         const float* bias, int E, int normalize, float* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && kv_len && proj && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && E > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        DeviceBuffer<float> pooled((size_t)n * w);
        kernels::text_head(x, kv_len, n, S, w, proj, bias, E, normalize, out, pooled.get(), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_cls_head(int device, const float* x, int n, int S, int w, const float* pool_w, const float* pool_b,
                        const float* cls_w, const float* cls_b, int L, int sigmoid, float* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && pool_w && pool_b && cls_w && cls_b && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && L > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::cls_head(x, S, n, w, pool_w, pool_b, cls_w, cls_b, L, sigmoid, out, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_owl_merge_ln(int device, const float* x, int n, int N, int w, const float* post_g, const float* post_b,
                            const float* det_g, const float* det_b, float eps, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && post_g && post_b && det_g && det_b && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && N >= 2 && w > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::owl_merge_ln(x, n, N, w, post_g, post_b, det_g, det_b, eps, static_cast<bf16*>(out), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_owl_class_logits(int device, const float* c, int ldc, int M, int E, const float* t, float* out,
                                void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(c && t && out, "NULL buffer");
        MB_CHECK_ARG(M > 0 && E > 0 && ldc >= E + 2, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::owl_class_logits(c, ldc, M, E, t, out, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_owl_boxes(int device, const void* a, int M, int w, int P, const float* w2, const float* b2,
                         const float* box_bias, float* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(a && w2 && b2 && box_bias && out, "NULL buffer");
        MB_CHECK_ARG(M > 0 && w > 0 && w % 4 == 0 && P > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::owl_boxes(static_cast<const bf16*>(a), M, w, P, w2, b2, box_bias, out, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_owl_box_bias(int G, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(out != nullptr, "NULL buffer");
        MB_CHECK_ARG(G > 0 && G <= 1024, "grid %d out of range", G);
        kernels::owl_box_bias(G, out);
    });
}

int b200_debug_frame_mean_head(int device, const float* x, int N, int T, const int32_t* row_in_seq, const float* gamma,
                               const float* beta, float eps, const float* proj, int n, int w, int E, float scale,
                               int normalize, float* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && gamma && beta && proj && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && N > 0 && T > 0 && w > 0 && E > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        DeviceBuffer<float> pooled((size_t)n * w);
        kernels::frame_mean_head(x, N, T, row_in_seq, gamma, beta, eps, proj, n, w, E, scale, normalize, out,
                                 pooled.get(), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_temporal_embed_ln(int device, float* x, const float* temb, int N, int T, const float* gamma,
                                 const float* beta, float eps, int rows, int w, void* h, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && gamma && beta && h, "NULL buffer");
        MB_CHECK_ARG(rows > 0 && N > 0 && T > 0 && w > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::temporal_embed_ln(x, temb, N, T, gamma, beta, eps, rows, w, static_cast<bf16*>(h), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_temporal_attention(int device, const void* qkv, int n, int T, int N, int W, int H, void* out,
                                  void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(qkv && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && N > 0, "n and N must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::temporal_attention(static_cast<const bf16*>(qkv), n, T, N, W, H, static_cast<bf16*>(out), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_temporal_attention_time(int device, int n, int T, int N, int W, int H, int iters, float* out_ms) {
    return guarded([&] {
        MB_CHECK_ARG(out_ms && n > 0 && N > 0 && iters > 0, "bad argument");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const long long rows = (long long)n * T * N;
        bf16* qkv = sc.alloc<bf16>((size_t)rows * 3 * W);
        bf16* o = sc.alloc<bf16>((size_t)rows * W);
        fill_bf16_kernel<<<(unsigned)((rows * 3 * W + 255) / 256), 256, 0, sc.s>>>(qkv, rows * 3 * W, 7u);
        MB_CUDA(cudaGetLastError());
        kernels::temporal_attention(qkv, n, T, N, W, H, o, sc.s);   // warm-up
        UniqueEvent e0 = make_event(), e1 = make_event();
        MB_CUDA(cudaEventRecord(e0.get(), sc.s));
        for (int i = 0; i < iters; ++i) kernels::temporal_attention(qkv, n, T, N, W, H, o, sc.s);
        MB_CUDA(cudaEventRecord(e1.get(), sc.s));
        MB_CUDA(cudaEventSynchronize(e1.get()));
        float ms = 0.f;
        MB_CUDA(cudaEventElapsedTime(&ms, e0.get(), e1.get()));
        *out_ms = ms / iters;
    });
}

int b200_debug_video_resize_crop(int device, const uint8_t* frames_hwc, int frames, int h, int w, int S,
                                 const float* mean3, const float* std3, float* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(frames_hwc && mean3 && std3 && out, "NULL buffer");
        MB_CHECK_ARG(frames > 0 && h > 0 && w > 0 && S > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::video_resize_crop(frames_hwc, frames, h, w, S, mean3, std3, out, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_l2_rows(int device, const float* src, int n, int E, int normalize, float* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(src && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && E > 0, "n, E must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::l2_rows(src, n, E, normalize, out, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_stem_im2col(int device, const uint8_t* hwc, const float* chw, int n, int S, const float* mean3,
                           const float* std3, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG((hwc != nullptr) != (chw != nullptr), "exactly one of hwc and chw");
        MB_CHECK_ARG(mean3 && std3 && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && S % 2 == 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::stem_im2col(hwc, chw, n, S, mean3, std3, static_cast<bf16*>(out), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_avgpool2(int device, const void* x, int n, int H, int W, int C, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && H > 0 && W > 0 && C > 0, "n, H, W, C must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::avgpool2_nhwc(static_cast<const bf16*>(x), n, H, W, C, static_cast<bf16*>(out), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_attnpool_tokens(int device, const void* x, const float* pos, int n, int HW, int C, void* out,
                               void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && pos && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && HW > 0 && C > 0, "n, HW, C must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::attnpool_tokens(static_cast<const bf16*>(x), pos, n, HW, C, static_cast<bf16*>(out), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_im2col_f32(int device, const float* chw, int n, int S, int p, int kpad, int cls, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(chw && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && p > 0 && S % p == 0 && S > 0 && (cls == 0 || cls == 1), "bad shape");
        MB_CHECK_ARG(kpad % 8 == 0 && kpad >= 3 * p * p, "kpad %d must be a multiple of 8 and >= 3 p^2", kpad);
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::im2col_f32(chw, n, S, p, kpad, cls, static_cast<bf16*>(out), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_resize(int device, const uint8_t* hwc, int n, int h, int w, int S, uint8_t* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(hwc && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && h > 0 && w > 0 && S > 0, "n, h, w, S must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::resize_crop_u8(hwc, n, h, w, S, out, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_resize_squash(int device, const uint8_t* hwc, int n, int h, int w, int S, uint8_t* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(hwc && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && h > 0 && w > 0 && S > 0, "n, h, w, S must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::resize_squash_u8(hwc, n, h, w, S, out, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_resize_ragged(int device, const uint8_t* const* d_hwc, const int32_t* heights, const int32_t* widths,
                             int n, int S, int squash, uint8_t* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(d_hwc && heights && widths && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0, "n, S must be positive");
        for (int i = 0; i < n; ++i) {
            MB_CHECK_ARG(d_hwc[i] != nullptr, "image %d is NULL", i);
            MB_CHECK_ARG(heights[i] > 0 && widths[i] > 0, "image %d: height %d and width %d must be positive", i,
                         heights[i], widths[i]);
        }
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::resize_u8(d_hwc, heights, widths, n, S, squash != 0, out, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_map_attention(int device, const float* q, int q_stride, const void* kv, int B, int S, int W, int H,
                             void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(q && kv && out, "NULL buffer");
        MB_CHECK_ARG(B > 0 && S > 0 && W > 0 && H > 0, "B, S, W, H must be positive");
        MB_CHECK_ARG(W == H * 64 || W == H * 96, "head_dim must be 64 or 96 (W %d, H %d)", W, H);
        MB_CHECK_ARG(q_stride == 0 || q_stride == W, "q_stride %d must be 0 or W %d", q_stride, W);
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::map_attention(q, q_stride, static_cast<const bf16*>(kv), B, S, W, H, static_cast<bf16*>(out), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_conv2d(int device, const void* x, int n, int H, int W, int cin, const float* w, int cout, int k,
                      const float* bias, const void* residual, int relu, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && w && bias && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && H > 0 && W > 0 && cout > 0, "n, H, W, cout must be positive");
        MB_CHECK_ARG(cin == 3 ? k == 3 && H == W && H % 2 == 0 : (k == 1 || (k == 3 && H == W)),
                     "unsupported conv: cin %d, k %d, %d x %d", cin, k, H, W);
        MB_CHECK_ARG(relu || !residual, "a residual needs the ReLU");
        MB_CHECK_ARG(relu || k == 1 || cin == 3, "the 3 x 3 gather conv runs with ReLU only");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        // the weight rows as the model's finalize lays them out, rounded to bf16 (nearest even) on the host
        std::vector<float> rows((size_t)cout * gemm::conv_rows_k(cin, k));
        gemm::conv_weight_rows(w, cout, cin, k, nullptr, rows.data());
        std::vector<bf16> rows_bf16(rows.size());
        std::transform(rows.begin(), rows.end(), rows_bf16.begin(), [](float v) { return __float2bfloat16_rn(v); });
        DeviceBuffer<bf16> dW(rows_bf16.size());
        MB_CUDA(cudaMemcpyAsync(dW.get(), rows_bf16.data(), rows_bf16.size() * sizeof(bf16), cudaMemcpyHostToDevice, s));
        const int Ho = cin == 3 ? H / 2 : H, Wo = cin == 3 ? W / 2 : W;
        gemm::Epilogue e;
        e.bias = bias;
        e.act = relu ? gemm::ACT_RELU : gemm::ACT_NONE;
        e.residual = residual;
        e.ldr = cout;
        e.out = out;
        e.ldo = cout;
        const bf16* a = static_cast<const bf16*>(x);
        DeviceBuffer<bf16> stem;
        if (cin == 3) {   // the stem: from already-normalised fp32 CHW, as b200_model_encode_images_f32 runs it
            stem = DeviceBuffer<bf16>((size_t)n * Ho * Wo * 64);
            const float mean[3] = {0.f, 0.f, 0.f}, std1[3] = {1.f, 1.f, 1.f};
            kernels::stem_im2col(nullptr, static_cast<const float*>(x), n, H, mean, std1, stem.get(), s);
            a = stem.get();
        }
        gemm::launch_conv(a, n, Ho, Wo, cin, k, dW.get(), cout, e, sm_count(device), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_dwconv7_ln(int device, const float* x, int n, int H, int W, int C, const float* w, const float* bias,
                          const float* gamma, const float* beta, float eps, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && w && bias && gamma && beta && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && H > 0 && W > 0 && C > 0, "n, H, W, C must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::dwconv7_ln(x, n, H, W, C, w, bias, gamma, beta, eps, static_cast<bf16*>(out), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_ln_pixels(int device, const float* x, int n, int H, int W, int C, const float* gamma, const float* beta,
                         float eps, int patchify, void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && gamma && beta && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && H > 0 && W > 0 && C > 0, "n, H, W, C must be positive");
        MB_CHECK_ARG(!patchify || (H % 2 == 0 && W % 2 == 0), "patchify needs an even H and W");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::ln_pixels(x, n, H, W, C, gamma, beta, eps, patchify ? nullptr : static_cast<float*>(out),
                           patchify ? static_cast<bf16*>(out) : nullptr, s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

int b200_debug_pool_ln(int device, const float* x, int n, int HW, int C, const float* gamma, const float* beta, float eps,
                       void* out, void* stream) {
    return guarded([&] {
        MB_CHECK_ARG(x && gamma && beta && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && HW > 0 && C > 0, "n, HW, C must be positive");
        require_device(device);
        DeviceGuard g(device);
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        kernels::pool_ln(x, n, HW, C, gamma, beta, eps, static_cast<bf16*>(out), s);
        MB_CUDA(cudaStreamSynchronize(s));
    });
}

}  // extern "C"
