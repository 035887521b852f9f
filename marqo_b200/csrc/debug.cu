// Diagnostic entry points: run one encoder kernel on host data (kernel-level numerics tests).
#include <vector>

#include "attention.cuh"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.cuh"
#include "score.cuh"

using namespace mb;

namespace {

struct Scratch {   // a stream and the device buffers of one call
    UniqueStream stream = make_stream(cudaStreamDefault);
    cudaStream_t s = stream.get();
    std::vector<DeviceBuffer<uint8_t>> bufs;
    template <class T>
    T* alloc(size_t n) {
        bufs.emplace_back(std::max<size_t>(n * sizeof(T), 16));
        return reinterpret_cast<T*>(bufs.back().get());
    }
    template <class T>
    T* upload(const T* h, size_t n) {
        T* d = alloc<T>(n);
        MB_CUDA(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
        return d;
    }
    __nv_bfloat16* upload_bf16(const float* h, size_t n) {
        float* f = upload(h, n);
        __nv_bfloat16* b = alloc<__nv_bfloat16>(n);
        kernels::f32_to_bf16(f, b, (long long)n, s);
        return b;
    }
};

__global__ void bf16_to_f32_kernel(const __nv_bfloat16* src, float* dst, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = __bfloat162float(src[i]);
}

// Runs `launch` (which writes bf16 [m] into its argument) and downloads the result as fp32.
template <class F>
void run_bf16_out(Scratch& sc, size_t m, float* out, F&& launch) {
    __nv_bfloat16* dO = sc.alloc<__nv_bfloat16>(m);
    float* dOut = sc.alloc<float>(m);
    launch(dO);
    bf16_to_f32_kernel<<<(unsigned)((m + 255) / 256), 256, 0, sc.s>>>(dO, dOut, (long long)m);
    MB_CUDA(cudaGetLastError());
    MB_CUDA(cudaMemcpyAsync(out, dOut, m * 4, cudaMemcpyDeviceToHost, sc.s));
    MB_CUDA(cudaStreamSynchronize(sc.s));
}

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
                           const float* mean3, const float* std3, const float* cls, const float* pos, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(hwc && conv_w && mean3 && std3 && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && patch > 0 && S % patch == 0 && N > 0 && N % 32 == 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const int G = (S / patch) * (S / patch), K = 3 * patch * patch;
        uint8_t* dImg = sc.upload(hwc, (size_t)n * S * S * 3);
        float* dW = sc.upload(conv_w, (size_t)N * K);
        const std::vector<float> zeros((size_t)(G + 1) * N, 0.f);   // a missing cls / pos
        const float* dCls = sc.upload(cls ? cls : zeros.data(), (size_t)N);
        const float* dPos = sc.upload(pos ? pos : zeros.data(), (size_t)(G + 1) * N);
        __nv_bfloat16* dWg = sc.alloc<__nv_bfloat16>((size_t)N * gemm::patch_gather_k(patch));
        kernels::patch_weight_rows(dW, N, patch, gemm::patch_gather_kbpd(patch), dWg, sc.s);
        // as the ViT forward does: x = pos (+ cls), then the gather GEMM adds conv1 onto it in place
        float* dX = sc.alloc<float>((size_t)n * (G + 1) * N);
        kernels::vit_embed_rows(dX, dCls, dPos, n, G + 1, N, sc.s);
        gemm::Epilogue ep;
        ep.residual = dX;
        ep.ldr = N;
        ep.out = dX;
        ep.ldo = N;
        ep.out_fp32 = 1;
        gemm::PatchGather pg;
        pg.img = dImg;
        pg.n = n;
        pg.S = S;
        pg.patch = patch;
        for (int i = 0; i < 3; ++i) {
            pg.mean[i] = mean3[i];
            pg.std[i] = std3[i];
        }
        gemm::launch_patch_embed(pg, dWg, N, ep, sc.s);
        MB_CUDA(cudaMemcpyAsync(out, dX, (size_t)n * (G + 1) * N * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
    });
}

int b200_debug_gemm_ln(int device, const float* A, const float* W, const float* bias, const float* residual, int M, int N,
                       int K, const float* gamma, const float* beta, float eps, int in_place, int repeats, float* out_x,
                       float* out_ln) {
    return guarded([&] {
        MB_CHECK_ARG(A && W && gamma && beta && out_x && out_ln, "NULL buffer");
        MB_CHECK_ARG(M > 0 && N > 0 && K > 0 && repeats > 0, "M, N, K, repeats must be positive");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        __nv_bfloat16* dA = sc.upload_bf16(A, (size_t)M * K);
        __nv_bfloat16* dW = sc.upload_bf16(W, (size_t)N * K);
        float* dOut = sc.alloc<float>((size_t)M * N);
        __nv_bfloat16* dLnB = sc.alloc<__nv_bfloat16>((size_t)M * N);
        float* dLnF = sc.alloc<float>((size_t)M * N);
        gemm::Epilogue ep;
        ep.bias = bias ? sc.upload(bias, (size_t)N) : nullptr;
        ep.residual = residual ? sc.upload(residual, (size_t)M * N) : nullptr;
        ep.ldr = N;
        ep.ldo = N;
        ep.out = dOut;
        ep.out_fp32 = 1;
        const float* dGamma = sc.upload(gamma, (size_t)N);
        const float* dBeta = sc.upload(beta, (size_t)N);
        // the residual GEMM followed by the LayerNorm launch of the encoder layer loops (model.cu); in place = BERT's
        // post-LN, where the normalised rows replace the fp32 output
        for (int i = 0; i < repeats; ++i) {
            gemm::launch(dA, K, dW, M, N, K, ep, sm_count(device), sc.s);
            kernels::layernorm(dOut, N, dGamma, dBeta, eps, M, N, in_place ? dOut : nullptr, dLnB, sc.s);
        }
        const long long n = (long long)M * N;
        bf16_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, sc.s>>>(dLnB, dLnF, n);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaMemcpyAsync(out_x, dOut, (size_t)M * N * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaMemcpyAsync(out_ln, dLnF, (size_t)M * N * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
    });
}

int b200_debug_gemm(int device, const float* A, const float* W, const float* bias, const float* residual, int M, int N,
                    int K, int act, int out_bf16, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(A && W && out, "NULL buffer");
        MB_CHECK_ARG(M > 0 && N > 0 && K > 0, "M, N, K must be positive");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        __nv_bfloat16* dA = sc.upload_bf16(A, (size_t)M * K);
        __nv_bfloat16* dW = sc.upload_bf16(W, (size_t)N * K);
        float* dOut = sc.alloc<float>((size_t)M * N);
        gemm::Epilogue ep;
        ep.bias = bias ? sc.upload(bias, (size_t)N) : nullptr;
        ep.residual = residual ? sc.upload(residual, (size_t)M * N) : nullptr;
        ep.ldr = N;
        ep.act = act;
        ep.ldo = N;
        __nv_bfloat16* dOutB = nullptr;
        if (out_bf16) {
            dOutB = sc.alloc<__nv_bfloat16>((size_t)M * N);
            ep.out = dOutB;
            ep.out_fp32 = 0;
        } else {
            ep.out = dOut;
            ep.out_fp32 = 1;
        }
        gemm::launch(dA, K, dW, M, N, K, ep, sm_count(device), sc.s);
        if (out_bf16) {
            const long long n = (long long)M * N;
            bf16_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, sc.s>>>(dOutB, dOut, n);
        }
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(sc.s));
        MB_CUDA(cudaMemcpy(out, dOut, (size_t)M * N * 4, cudaMemcpyDeviceToHost));
    });
}

int b200_debug_gemm_into(int device, const float* A, const float* W, const float* bias, int M, int N, int K, int act,
                         int out_bf16, int residual_in_place, int out_rows, int ldo, int sms, float* io,
                         int* kernel_out) {
    return guarded([&] {
        MB_CHECK_ARG(A && W && io, "NULL buffer");
        MB_CHECK_ARG(M > 0 && N > 0 && K > 0 && out_rows >= M && ldo >= N && sms >= 0, "bad shape");
        MB_CHECK_ARG(!(residual_in_place && out_bf16), "the in-place residual is fp32");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        __nv_bfloat16* dA = sc.upload_bf16(A, (size_t)M * K);
        __nv_bfloat16* dW = sc.upload_bf16(W, (size_t)N * K);
        const size_t n = (size_t)out_rows * ldo;
        float* dIo = sc.upload(io, n);
        __nv_bfloat16* dIoB = out_bf16 ? sc.upload_bf16(io, n) : nullptr;
        gemm::Epilogue ep;
        ep.bias = bias ? sc.upload(bias, (size_t)N) : nullptr;
        ep.act = act;
        ep.out = out_bf16 ? static_cast<void*>(dIoB) : static_cast<void*>(dIo);
        ep.ldo = ldo;
        ep.out_fp32 = out_bf16 ? 0 : 1;
        if (residual_in_place) {   // as the encoder layers update the fp32 residual stream: residual == out
            ep.residual = dIo;
            ep.ldr = ldo;
        }
        const int kernel = gemm::launch(dA, K, dW, M, N, K, ep, sms > 0 ? sms : sm_count(device), sc.s);
        if (kernel_out) *kernel_out = kernel;
        if (out_bf16) bf16_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, sc.s>>>(dIoB, dIo, (long long)n);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(sc.s));
        MB_CUDA(cudaMemcpy(io, dIo, n * 4, cudaMemcpyDeviceToHost));
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

int b200_debug_attention(int device, const float* qkv, int B, int S, int W, int H, int mask, const int32_t* kv_len,
                         const float* rel_bias, int smax, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(qkv && out, "NULL buffer");
        MB_CHECK_ARG(B > 0 && S > 0 && W > 0 && H > 0, "B, S, W, H must be positive");
        MB_CHECK_ARG(!rel_bias || smax > 0, "smax must be positive");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const size_t M = (size_t)B * S;
        __nv_bfloat16* dq = sc.upload_bf16(qkv, M * 3 * W);
        __nv_bfloat16* dO = sc.alloc<__nv_bfloat16>(M * W);
        float* dOut = sc.alloc<float>(M * W);
        const int32_t* dlen = kv_len ? sc.upload(kv_len, (size_t)B) : nullptr;
        attention::RelBias bias;
        if (rel_bias) {
            const size_t span = (size_t)H * (2 * smax - 1);
            std::vector<float> scaled(rel_bias, rel_bias + span);   // the kernels add it in the log2 domain
            for (float& v : scaled) v *= 1.4426950408889634f;
            bias.table = sc.upload(scaled.data(), span);
            bias.smax = smax;
        }
        attention::launch(dq, dO, B, S, W, H, mask, dlen, bias, sc.s);
        const long long n = (long long)M * W;
        bf16_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, sc.s>>>(dO, dOut, n);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(sc.s));
        MB_CUDA(cudaMemcpy(out, dOut, M * W * 4, cudaMemcpyDeviceToHost));
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
        std::vector<int32_t> lens((size_t)B, S);
        const int32_t* dlen = mask == attention::MASK_KEYLEN ? sc.upload(lens.data(), (size_t)B) : nullptr;
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
                         int rows, int w, int in_place, float* out_f32, float* out_bf16) {
    return guarded([&] {
        MB_CHECK_ARG(x && gamma && beta && (out_f32 || out_bf16), "NULL buffer");
        MB_CHECK_ARG(rows > 0 && w > 0 && in_stride >= 0, "rows, w must be positive");
        if (in_stride == 0) in_stride = w;
        MB_CHECK_ARG(in_stride >= w, "in_stride %lld < w %d", in_stride, w);
        MB_CHECK_ARG(!in_place || (out_f32 && in_stride == w), "in place needs the fp32 output and compact rows");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        float* dx = sc.upload(x, (size_t)(rows - 1) * in_stride + w);
        float* dg = sc.upload(gamma, (size_t)w);
        float* db = sc.upload(beta, (size_t)w);
        const size_t n = (size_t)rows * w;
        float* dF = out_f32 ? (in_place ? dx : sc.alloc<float>(n)) : nullptr;
        __nv_bfloat16* dB = out_bf16 ? sc.alloc<__nv_bfloat16>(n) : nullptr;
        kernels::layernorm(dx, in_stride, dg, db, eps, rows, w, dF, dB, sc.s);
        if (dB) {
            float* dBf = sc.alloc<float>(n);
            bf16_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, sc.s>>>(dB, dBf, (long long)n);
            MB_CUDA(cudaGetLastError());
            MB_CUDA(cudaMemcpyAsync(out_bf16, dBf, n * 4, cudaMemcpyDeviceToHost, sc.s));
        }
        if (dF) MB_CUDA(cudaMemcpyAsync(out_f32, dF, n * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
    });
}

int b200_debug_clip_text_embed(int device, const int32_t* ids, const float* tok, const float* pos, int n, int S, int w,
                               int vocab, float* x, int32_t* eot) {
    return guarded([&] {
        MB_CHECK_ARG(ids && tok && pos && x && eot, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && w % 4 == 0 && vocab > 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const size_t rows = (size_t)n * S;
        const int32_t* dIds = sc.upload(ids, rows);
        const float* dTok = sc.upload(tok, (size_t)vocab * w);
        const float* dPos = sc.upload(pos, (size_t)S * w);
        float* dX = sc.alloc<float>(rows * w);
        int32_t* dEot = sc.alloc<int32_t>((size_t)n);
        kernels::clip_text_embed(dIds, dTok, dPos, n, S, w, vocab, dX, dEot, sc.s);
        MB_CUDA(cudaMemcpyAsync(x, dX, rows * w * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaMemcpyAsync(eot, dEot, (size_t)n * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
    });
}

// The BERT and RoBERTa embedding hooks: pos has pos_rows rows, which must cover every position the kernel reads.
static int debug_embed_ln(int device, bool roberta, const int32_t* ids, const int32_t* mask, const float* word,
                          const float* pos, int pos_rows, const float* type0, const float* gamma, const float* beta,
                          float eps, int n, int S, int w, int vocab, int pad, float* x, float* h, int32_t* kv_len) {
    return guarded([&] {
        MB_CHECK_ARG(ids && word && pos && gamma && beta && x && h && kv_len, "NULL buffer");
        MB_CHECK_ARG(roberta || type0, "the BERT embedding always adds token-type row 0");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && vocab > 0, "bad shape");
        MB_CHECK_ARG(roberta ? pad >= 0 && pos_rows >= pad + S + 1 : pos_rows >= S, "%d position rows are too few",
                     pos_rows);
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const size_t rows = (size_t)n * S;
        const int32_t* dIds = sc.upload(ids, rows);
        const int32_t* dMask = mask ? sc.upload(mask, rows) : nullptr;
        const float* dWord = sc.upload(word, (size_t)vocab * w);
        const float* dPos = sc.upload(pos, (size_t)pos_rows * w);
        const float* dType = type0 ? sc.upload(type0, (size_t)w) : nullptr;
        const float* dG = sc.upload(gamma, (size_t)w);
        const float* dB = sc.upload(beta, (size_t)w);
        float* dX = sc.alloc<float>(rows * w);
        __nv_bfloat16* dH = sc.alloc<__nv_bfloat16>(rows * w);
        float* dHf = sc.alloc<float>(rows * w);
        int32_t* dLen = sc.alloc<int32_t>((size_t)n);
        if (roberta)
            kernels::roberta_embed_ln(dIds, dMask, dWord, dPos, dType, dG, dB, eps, n, S, w, vocab, pad, dX, dH, dLen, sc.s);
        else
            kernels::bert_embed_ln(dIds, dMask, dWord, dPos, dType, dG, dB, eps, n, S, w, vocab, dX, dH, dLen, sc.s);
        const long long m = (long long)(rows * w);
        bf16_to_f32_kernel<<<(unsigned)((m + 255) / 256), 256, 0, sc.s>>>(dH, dHf, m);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaMemcpyAsync(x, dX, rows * w * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaMemcpyAsync(h, dHf, rows * w * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaMemcpyAsync(kv_len, dLen, (size_t)n * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
    });
}

int b200_debug_bert_embed_ln(int device, const int32_t* ids, const int32_t* mask, const float* word, const float* pos,
                             int pos_rows, const float* type0, const float* gamma, const float* beta, float eps, int n,
                             int S, int w, int vocab, float* x, float* h, int32_t* kv_len) {
    return debug_embed_ln(device, false, ids, mask, word, pos, pos_rows, type0, gamma, beta, eps, n, S, w, vocab, 0, x, h,
                          kv_len);
}

int b200_debug_roberta_embed_ln(int device, const int32_t* ids, const int32_t* mask, const float* word, const float* pos,
                                int pos_rows, const float* type0, const float* gamma, const float* beta, float eps, int n,
                                int S, int w, int vocab, int pad, float* x, float* h, int32_t* kv_len) {
    return debug_embed_ln(device, true, ids, mask, word, pos, pos_rows, type0, gamma, beta, eps, n, S, w, vocab, pad, x,
                          h, kv_len);
}

int b200_debug_clip_head(int device, const float* x, int S, const int32_t* row_in_seq, const float* gamma,
                         const float* beta, float eps, const float* proj, int n, int w, int E, int normalize, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(x && gamma && beta && proj && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && E > 0, "bad shape");
        for (int b = 0; row_in_seq && b < n; ++b)
            MB_CHECK_ARG(row_in_seq[b] >= 0 && row_in_seq[b] < S, "row_in_seq[%d] = %d outside [0, %d)", b, row_in_seq[b], S);
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const float* dX = sc.upload(x, (size_t)n * S * w);
        const int32_t* dRow = row_in_seq ? sc.upload(row_in_seq, (size_t)n) : nullptr;
        const float* dG = sc.upload(gamma, (size_t)w);
        const float* dB = sc.upload(beta, (size_t)w);
        const float* dP = sc.upload(proj, (size_t)w * E);
        float* dOut = sc.alloc<float>((size_t)n * E);
        float* dPooled = sc.alloc<float>((size_t)n * w);
        kernels::clip_head(dX, S, dRow, dG, dB, eps, dP, n, w, E, normalize, dOut, dPooled, sc.s);
        MB_CUDA(cudaMemcpyAsync(out, dOut, (size_t)n * E * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
    });
}

int b200_debug_bert_head(int device, const float* x, const int32_t* kv_len, int n, int S, int w, int pool, int normalize,
                         float* out) {
    return guarded([&] {
        MB_CHECK_ARG(x && kv_len && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && w > 0 && (pool == 0 || pool == 1), "bad shape or pool");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const float* dX = sc.upload(x, (size_t)n * S * w);
        const int32_t* dLen = sc.upload(kv_len, (size_t)n);
        float* dOut = sc.alloc<float>((size_t)n * w);
        kernels::bert_head(dX, dLen, n, S, w, pool, normalize, dOut, sc.s);
        MB_CUDA(cudaMemcpyAsync(out, dOut, (size_t)n * w * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
    });
}

int b200_debug_l2_rows(int device, const float* src, int n, int E, int normalize, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(src && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && E > 0, "n, E must be positive");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const float* dS = sc.upload(src, (size_t)n * E);
        float* dOut = sc.alloc<float>((size_t)n * E);
        kernels::l2_rows(dS, n, E, normalize, dOut, sc.s);
        MB_CUDA(cudaMemcpyAsync(out, dOut, (size_t)n * E * 4, cudaMemcpyDeviceToHost, sc.s));
        MB_CUDA(cudaStreamSynchronize(sc.s));
    });
}

int b200_debug_stem_im2col(int device, const uint8_t* hwc, const float* chw, int n, int S, const float* mean3,
                           const float* std3, float* out) {
    return guarded([&] {
        MB_CHECK_ARG((hwc != nullptr) != (chw != nullptr), "exactly one of hwc and chw");
        MB_CHECK_ARG(mean3 && std3 && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && S > 0 && S % 2 == 0, "bad shape");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const size_t px = (size_t)n * S * S * 3;
        const uint8_t* dU8 = hwc ? sc.upload(hwc, px) : nullptr;
        const float* dChw = chw ? sc.upload(chw, px) : nullptr;
        run_bf16_out(sc, (size_t)n * (S / 2) * (S / 2) * 64, out, [&](__nv_bfloat16* o) {
            kernels::stem_im2col(dU8, dChw, n, S, mean3, std3, o, sc.s);
        });
    });
}

int b200_debug_avgpool2(int device, const float* x, int n, int H, int W, int C, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(x && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && H > 0 && W > 0 && C > 0, "n, H, W, C must be positive");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const __nv_bfloat16* dX = sc.upload_bf16(x, (size_t)n * H * W * C);
        run_bf16_out(sc, (size_t)n * (H / 2) * (W / 2) * C, out,
                     [&](__nv_bfloat16* o) { kernels::avgpool2_nhwc(dX, n, H, W, C, o, sc.s); });
    });
}

int b200_debug_attnpool_tokens(int device, const float* x, const float* pos, int n, int HW, int C, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(x && pos && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && HW > 0 && C > 0, "n, HW, C must be positive");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const __nv_bfloat16* dX = sc.upload_bf16(x, (size_t)n * HW * C);
        const float* dPos = sc.upload(pos, (size_t)(HW + 1) * C);
        run_bf16_out(sc, (size_t)n * (HW + 1) * C, out,
                     [&](__nv_bfloat16* o) { kernels::attnpool_tokens(dX, dPos, n, HW, C, o, sc.s); });
    });
}

int b200_debug_im2col_f32(int device, const float* chw, int n, int S, int p, int kpad, int cls, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(chw && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && p > 0 && S % p == 0 && S > 0 && (cls == 0 || cls == 1), "bad shape");
        MB_CHECK_ARG(kpad % 8 == 0 && kpad >= 3 * p * p, "kpad %d must be a multiple of 8 and >= 3 p^2", kpad);
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const float* dChw = sc.upload(chw, (size_t)n * 3 * S * S);
        const int g2 = (S / p) * (S / p);
        run_bf16_out(sc, (size_t)n * (g2 + cls) * kpad, out,
                     [&](__nv_bfloat16* o) { kernels::im2col_f32(dChw, n, S, p, kpad, cls, o, sc.s); });
    });
}

int b200_debug_resize(int device, const uint8_t* hwc, int n, int h, int w, int S, uint8_t* out) {
    return guarded([&] {
        MB_CHECK_ARG(hwc && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && h > 0 && w > 0 && S > 0, "n, h, w, S must be positive");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        uint8_t* din = sc.upload(hwc, (size_t)n * h * w * 3);
        uint8_t* dout = sc.alloc<uint8_t>((size_t)n * S * S * 3);
        kernels::resize_crop_u8(din, n, h, w, S, dout, sc.s);
        MB_CUDA(cudaStreamSynchronize(sc.s));
        MB_CUDA(cudaMemcpy(out, dout, (size_t)n * S * S * 3, cudaMemcpyDeviceToHost));
    });
}

int b200_debug_resize_squash(int device, const uint8_t* hwc, int n, int h, int w, int S, uint8_t* out) {
    return guarded([&] {
        MB_CHECK_ARG(hwc && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && h > 0 && w > 0 && S > 0, "n, h, w, S must be positive");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        uint8_t* din = sc.upload(hwc, (size_t)n * h * w * 3);
        uint8_t* dout = sc.alloc<uint8_t>((size_t)n * S * S * 3);
        kernels::resize_squash_u8(din, n, h, w, S, dout, sc.s);
        MB_CUDA(cudaStreamSynchronize(sc.s));
        MB_CUDA(cudaMemcpy(out, dout, (size_t)n * S * S * 3, cudaMemcpyDeviceToHost));
    });
}

static int debug_map_attention(int device, const float* q, bool per_image, const float* kv, int B, int S, int W, int H,
                               float* out) {
    return guarded([&] {
        MB_CHECK_ARG(q && kv && out, "NULL buffer");
        MB_CHECK_ARG(B > 0 && S > 0 && W > 0 && H > 0, "B, S, W, H must be positive");
        MB_CHECK_ARG(W == H * 64, "head_dim must be 64 (W %d, H %d)", W, H);
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const size_t M = (size_t)B * S;
        const float* dq = sc.upload(q, (size_t)W * (per_image ? B : 1));
        __nv_bfloat16* dkv = sc.upload_bf16(kv, M * 2 * W);
        __nv_bfloat16* dO = sc.alloc<__nv_bfloat16>((size_t)B * W);
        float* dOut = sc.alloc<float>((size_t)B * W);
        kernels::map_attention(dq, per_image ? W : 0, dkv, B, S, W, H, dO, sc.s);
        const long long n = (long long)B * W;
        bf16_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, sc.s>>>(dO, dOut, n);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(sc.s));
        MB_CUDA(cudaMemcpy(out, dOut, (size_t)B * W * 4, cudaMemcpyDeviceToHost));
    });
}

int b200_debug_map_attention(int device, const float* q, const float* kv, int B, int S, int W, int H, float* out) {
    return debug_map_attention(device, q, false, kv, B, S, W, H, out);
}

int b200_debug_map_attention_per_image(int device, const float* q, const float* kv, int B, int S, int W, int H,
                                       float* out) {
    return debug_map_attention(device, q, true, kv, B, S, W, H, out);
}

int b200_debug_conv2d(int device, const float* x, int n, int H, int W, int cin, const float* w, int cout, int k,
                      const float* bias, const float* residual, int relu, float* out) {
    return guarded([&] {
        MB_CHECK_ARG(x && w && out, "NULL buffer");
        MB_CHECK_ARG(n > 0 && H > 0 && W > 0 && cout > 0, "n, H, W, cout must be positive");
        MB_CHECK_ARG(cin == 3 ? k == 3 && H == W && H % 2 == 0 : (k == 1 || (k == 3 && H == W)),
                     "unsupported conv: cin %d, k %d, %d x %d", cin, k, H, W);
        MB_CHECK_ARG(relu || !residual, "a residual needs the ReLU");
        MB_CHECK_ARG(relu || k == 1 || cin == 3, "the 3 x 3 gather conv runs with ReLU only");
        require_device(device);
        DeviceGuard g(device);
        Scratch sc;
        const int K = gemm::conv_rows_k(cin, k);
        std::vector<float> rows((size_t)cout * K);
        gemm::conv_weight_rows(w, cout, cin, k, nullptr, rows.data());
        __nv_bfloat16* dW = sc.upload_bf16(rows.data(), rows.size());
        std::vector<float> zeros;
        if (!bias) zeros.assign((size_t)cout, 0.f);
        const float* dB = sc.upload(bias ? bias : zeros.data(), (size_t)cout);
        const int Ho = cin == 3 ? H / 2 : H, Wo = cin == 3 ? W / 2 : W;
        const size_t out_n = (size_t)n * Ho * Wo * cout;
        gemm::Epilogue e;
        e.bias = dB;
        e.act = relu ? gemm::ACT_RELU : gemm::ACT_NONE;
        e.residual = residual ? sc.upload_bf16(residual, out_n) : nullptr;
        e.ldr = cout;
        __nv_bfloat16* dO = sc.alloc<__nv_bfloat16>(out_n);
        e.out = dO;
        e.ldo = cout;
        const __nv_bfloat16* dX;
        if (cin == 3) {   // the stem: from already-normalised fp32 CHW, as b200_model_encode_images_f32 runs it
            std::vector<float> chw((size_t)n * 3 * H * W);
            for (int b = 0; b < n; ++b)
                for (int c = 0; c < 3; ++c)
                    for (int i = 0; i < H * W; ++i) chw[((size_t)b * 3 + c) * H * W + i] = x[((size_t)b * H * W + i) * 3 + c];
            const float* dchw = sc.upload(chw.data(), chw.size());
            __nv_bfloat16* dA = sc.alloc<__nv_bfloat16>((size_t)n * Ho * Wo * 64);
            const float mean[3] = {0.f, 0.f, 0.f}, std1[3] = {1.f, 1.f, 1.f};
            kernels::stem_im2col(nullptr, dchw, n, H, mean, std1, dA, sc.s);
            dX = dA;
        } else {
            dX = sc.upload_bf16(x, (size_t)n * H * W * cin);
        }
        gemm::launch_conv(dX, n, Ho, Wo, cin, k, dW, cout, e, sm_count(device), sc.s);
        float* dOut = sc.alloc<float>(out_n);
        bf16_to_f32_kernel<<<(unsigned)((out_n + 255) / 256), 256, 0, sc.s>>>(dO, dOut, (long long)out_n);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(sc.s));
        MB_CUDA(cudaMemcpy(out, dOut, out_n * 4, cudaMemcpyDeviceToHost));
    });
}

}  // extern "C"
