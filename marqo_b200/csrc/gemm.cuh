// Warp-specialised wgmma GEMM:  out[M,N] = epilogue( A[M,K] (bf16, K-major) x W[N,K]^T (bf16, K-major) )
// 128 x 128 tiles, TMA-fed 128B-swizzled smem ring, two MMA warpgroups with fp32 accumulators in registers.  For
// K >= 1024, N % 256 == 0 and at least one full wave of tiles, a persistent kernel of 128 x 256 tiles (one CTA per SM)
// runs instead.  Both kernels run one epilogue, act(acc + bias) (+ residual): each warpgroup's output block goes
// through shared memory (the fp32 residual TMA-loaded into it ahead of time) and out by TMA stores (gemm.cu).
// Output and residual must be 16-byte aligned; a residual needs an fp32 output and ldr % 4 == 0, or ACT_RELU (bf16
// output) and ldr % 8 == 0.
#pragma once
#include "common.cuh"

namespace mb {
namespace gemm {

// ACT_RELU: bf16 output only; its residual (bf16 [M, ldr]) is added before the activation: relu(acc + bias + residual),
// the ResNet bottleneck's ReLU(out + identity).
enum Act { ACT_NONE = 0, ACT_GELU = 1, ACT_QUICKGELU = 2, ACT_RELU = 3 };

struct Epilogue {
    const float* bias = nullptr;      // [N]
    const void* residual = nullptr;   // fp32 [M, ldr], added after the activation; bf16 before it with ACT_RELU
    int ldr = 0;
    int act = ACT_NONE;   // erf-GELU on packed fp16 pairs for a bf16 output (see gemm.cu gelu_erf_h2), fp32 otherwise
    void* out = nullptr;  // bf16 or fp32 [*, ldo]
    int ldo = 0;
    int out_fp32 = 0;
};

// A: bf16 [M, K] row-major with leading dimension lda (elements); W: bf16 [N, K] row-major (nn.Linear layout).
// Requirements: K % 8 == 0 (the last 64-wide k-block is zero-filled past K in A and W by TMA), N % 8 == 0 for a bf16
// output and N % 32 == 0 for an fp32 one (the last output box is clipped at N), lda % 8 == 0.
// Returns the kernel it launched: KERNEL_PERSISTENT for K >= 1024, K % 64 == 0, N % 256 == 0 and at least sm_count
// 128 x 256 tiles,
// KERNEL_128x128 otherwise, KERNEL_NONE when M or N is 0.
enum Kernel { KERNEL_NONE = -1, KERNEL_128x128 = 0, KERNEL_PERSISTENT = 1 };
int launch(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int M, int N, int K, const Epilogue& ep,
           int sm_count, cudaStream_t stream);

// ViT patch embedding straight from uint8 pixels (SURVEY §8 a2; add_docs.py:129-134 + clip_utils.py:48-67 fused into the
// conv1 GEMM's operand load): out = epilogue( patches(img) x Wg^T ) over the n (g^2 + cls) ViT token rows of the uint8
// HWC batch [n, S, S, 3] (S % patch == 0, g = S / patch).  Row r of the virtual A matrix is token t = r % (g^2 + cls)
// of image r / (g^2 + cls): zero for the class token t < cls, else patch t - cls (row-major in the g x g grid),
// normalised as ToTensor + Normalize.  cls is 1 for CLIP and 0 for the class-token-free SigLIP tower.  Wg [N,
// patch_gather_k(patch)] is conv1.weight re-laid by kernels::patch_weight_rows.  No patch matrix exists in HBM: the
// gather warps of the GEMM read the image rows, convert and write the swizzled smem A stage.  The epilogue must have an
// fp32 output and no activation.  Returns the number of kernels launched (0 without images, else 1).
struct PatchGather {
    const uint8_t* img = nullptr;
    int n = 0, S = 0, patch = 0;
    int cls = 1;
    float mean[3] = {0.f, 0.f, 0.f}, std[3] = {1.f, 1.f, 1.f};
};
inline int patch_gather_kbpd(int patch) { return (3 * patch + 63) / 64; }
inline int patch_gather_k(int patch) { return patch * patch_gather_kbpd(patch) * 64; }
int launch_patch_embed(const PatchGather& pg, const __nv_bfloat16* Wg, int N, const Epilogue& ep, cudaStream_t stream);

// 3 x 3 convolution, stride 1, zero padding 1, as an implicit GEMM over an NHWC bf16 activation [n, H, W, cin]:
// row r of the virtual A matrix is output pixel (b, y, x) = r in row-major order (a 128-row tile may span images), and
// its k index tap * cin + c, tap = 3 (dy + 1) + (dx + 1), reads input pixel (y + dy, x + dx), zero outside the image.
// The four gather warps of the GEMM copy 16-byte channel chunks into the swizzled A stage; k-block kb covers
// k = 64 kb .. 64 kb + 63 (part of a tap, or parts of several taps when cin is not a multiple of 64), and k >= 9 cin
// is zero.  W: bf16 [N, conv_gather_k(cin)] with the same k order (conv.weight [N, cin, 3, 3] permuted to
// [N, 3, 3, cin], zero padded).  cin and N must be multiples of 8 (the ResNets' 40 ... 768); out is the NHWC
// [n, H, W, N] output.  Returns the number of kernels launched.
struct ConvGather {
    const __nv_bfloat16* act = nullptr;
    int n = 0, H = 0, W = 0, cin = 0;
};
inline int conv_gather_k(int cin) { return (9 * cin + 63) / 64 * 64; }
int launch_conv3x3(const ConvGather& cg, const __nv_bfloat16* Wc, int N, const Epilogue& ep, cudaStream_t stream);

// The ResNet convolutions as the kernels run them: a k x k conv of cin channels has W rows of conv_rows_k(cin, k)
// columns: cin for a 1 x 1 conv (a GEMM over the NHWC pixel rows), conv_gather_k(cin) for a 3 x 3 (launch_conv3x3),
// 64 for the 3-channel stem conv (kernels::stem_im2col's k = tap * 3 + c).
int conv_rows_k(int cin, int k);
// One such conv over n images of H x W output pixels, x -> ep.out (NHWC bf16): a 3 x 3 conv (cin != 3) by
// launch_conv3x3, any other by launch over x's rows, the NHWC pixel rows of a 1 x 1 conv or kernels::stem_im2col's rows
// for the stem.  Wc: [cout, conv_rows_k(cin, k)] (conv_weight_rows).  Returns the number of kernels launched.
int launch_conv(const __nv_bfloat16* x, int n, int H, int W, int cin, int k, const __nv_bfloat16* Wc, int cout,
                const Epilogue& ep, int sms, cudaStream_t stream);
// Host: conv.weight fp32 [cout, cin, k, k] times scale[o] (NULL: 1; the folded BatchNorm), in double, -> fp32 rows
// [cout, conv_rows_k(cin, k)] with k index tap * cin + c (tap = k ky + kx), zero padded.
void conv_weight_rows(const float* w, int cout, int cin, int k, const double* scale, float* out);

void configure();  // one-time cudaFuncSetAttribute calls

}  // namespace gemm
}  // namespace mb
