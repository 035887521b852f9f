#include <algorithm>
#include <atomic>
#include <vector>

#include "common.cuh"

#include <mutex>

namespace mb {

static thread_local std::string g_last_error;
static std::atomic<int64_t> g_device_bytes{0};

void set_last_error(const std::string& msg) { g_last_error = msg; }

void require_sm90_device(int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        fail(B200_ERR_NO_DEVICE, "no CUDA device available (marqo_b200 has no CPU fallback)");
    }
    MB_CHECK_ARG(device >= 0 && device < ndev, "device %d out of range (%d devices)", device, ndev);
    int major = 0;
    MB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    if (major != 9) fail(B200_ERR_NO_DEVICE, "device %d has compute capability %d.x; sm_90 required", device, major);
}

void* device_alloc(size_t bytes, cudaStream_t stream, bool stream_ordered) {
    void* p = nullptr;
    const cudaError_t e = stream_ordered ? cudaMallocAsync(&p, bytes, stream) : cudaMalloc(&p, bytes);
    if (e == cudaErrorMemoryAllocation) {
        cudaGetLastError();
        fail(B200_ERR_OOM, "cudaMalloc(%zu bytes) failed: out of device memory", bytes);
    }
    if (e != cudaSuccess)
        fail(B200_ERR_CUDA, "%s(%zu bytes) failed: %s", stream_ordered ? "cudaMallocAsync" : "cudaMalloc", bytes,
             cudaGetErrorString(e));
    g_device_bytes += (int64_t)bytes;
    return p;
}

void device_free(void* p, size_t bytes, cudaStream_t stream, bool stream_ordered) noexcept {
    if (stream_ordered) cudaFreeAsync(p, stream);
    else cudaFree(p);
    g_device_bytes -= (int64_t)bytes;
}

UniqueStream make_stream(unsigned flags) {
    cudaStream_t s = nullptr;
    MB_CUDA(cudaStreamCreateWithFlags(&s, flags));
    return UniqueStream(s);
}

UniqueEvent make_event() {
    cudaEvent_t e = nullptr;
    MB_CUDA(cudaEventCreate(&e));
    return UniqueEvent(e);
}

void* pinned_alloc(size_t bytes) {
    void* p = nullptr;
    MB_CUDA(cudaHostAlloc(&p, bytes, cudaHostAllocPortable));
    return p;
}

IpcMapping open_ipc_mapping(const cudaIpcMemHandle_t& h) {
    void* p = nullptr;
    MB_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    return IpcMapping(static_cast<uint8_t*>(p));
}

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    if (!fn) fail(B200_ERR_NO_DEVICE, "cuTensorMapEncodeTiled is not available from the CUDA driver");
    return fn;
}

CUtensorMap make_tmap_2d(const void* base, CUtensorMapDataType dtype, uint32_t elem_bytes, uint64_t cols,
                         uint64_t rows, uint64_t row_pitch_bytes, uint32_t box_cols, uint32_t box_rows,
                         CUtensorMapSwizzle swizzle) {
    CUtensorMap tm;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {row_pitch_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estride[2] = {1, 1};
    (void)elem_bytes;
    CUresult r = encode_tiled_fn()(&tm, dtype, 2, const_cast<void*>(base), gdim, gstride, box, estride,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        fail(B200_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d): cols=%llu rows=%llu pitch=%llu box=%ux%u", (int)r,
             (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)row_pitch_bytes, box_cols,
             box_rows);
    return tm;
}

int sm_count(int device) {
    int n = 0;
    MB_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device));
    return n;
}

}  // namespace mb

extern "C" {

int b200_abi_version(void) { return B200_ABI_VERSION; }

const char* b200_last_error(void) { return mb::g_last_error.c_str(); }

int b200_device_count(int* out_count) {
    return mb::guarded([&] {
        MB_CHECK_ARG(out_count != nullptr, "out_count is NULL");
        int n = 0;
        cudaError_t e = cudaGetDeviceCount(&n);
        if (e != cudaSuccess) {
            cudaGetLastError();
            n = 0;
        }
        int ok = 0;
        for (int d = 0; d < n; ++d) {
            int major = 0;
            if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, d) == cudaSuccess && major == 9)
                ++ok;
        }
        *out_count = ok;
    });
}

int b200_host_alloc(size_t bytes, void** out) {
    return mb::guarded([&] {
        MB_CHECK_ARG(out != nullptr, "out is NULL");
        *out = nullptr;
        MB_CHECK_ARG(bytes > 0, "bytes must be positive");
        void* p = nullptr;
        const cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocPortable);
        if (e == cudaErrorMemoryAllocation) {
            cudaGetLastError();
            mb::fail(B200_ERR_OOM, "cudaHostAlloc(%zu bytes) failed: out of page-locked host memory", bytes);
        }
        if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) {
            cudaGetLastError();
            mb::fail(B200_ERR_NO_DEVICE, "no CUDA device available (marqo_b200 has no CPU fallback)");
        }
        MB_CUDA(e);
        *out = p;
    });
}

int b200_host_free(void* p) {
    return mb::guarded([&] {
        if (p) MB_CUDA(cudaFreeHost(p));
    });
}

int b200_debug_device_bytes(int64_t* out_live_bytes) {
    return mb::guarded([&] {
        MB_CHECK_ARG(out_live_bytes != nullptr, "out_live_bytes is NULL");
        *out_live_bytes = mb::g_device_bytes.load();
    });
}

int b200_fuse_vectors(const double* vecs, const double* weights, int n, int dim, int normalize, double* out) {
    return mb::guarded([&] {
        MB_CHECK_ARG(vecs && weights && out, "NULL argument");
        MB_CHECK_ARG(n > 0 && dim > 0, "n and dim must be positive");
        // np.mean([w_i * v_i], axis=0): pairwise order of numpy's add.reduce over axis 0 is sequential
        // for a short leading axis, so a plain left-to-right sum reproduces it.
        for (int d = 0; d < dim; ++d) {
            double acc = 0.0;
            for (int i = 0; i < n; ++i) acc += vecs[(size_t)i * dim + d] * weights[i];
            out[d] = acc / (double)n;
        }
        if (normalize) {
            double ss = 0.0;
            for (int d = 0; d < dim; ++d) ss += out[d] * out[d];
            double nrm = sqrt(ss);
            if (nrm > 0.0)
                for (int d = 0; d < dim; ++d) out[d] /= nrm;
        }
    });
}

namespace {

// One SLERP step of the reference (vector_interpolation.py:160-195): angle from the normalised dot product, linear
// fallback for co-linear inputs.  Returns false when either input has zero length.
bool slerp_pair(const double* v0, const double* v1, double t, int dim, double* out) {
    double dot = 0.0, n0 = 0.0, n1 = 0.0;
    for (int i = 0; i < dim; ++i) {
        dot += v0[i] * v1[i];
        n0 += v0[i] * v0[i];
        n1 += v1[i] * v1[i];
    }
    n0 = sqrt(n0);
    n1 = sqrt(n1);
    if (n0 == 0.0 || n1 == 0.0) return false;
    double c = dot / (n0 * n1);
    c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
    const double theta = acos(c);
    const double st = sin(theta);
    if (st == 0.0) {
        for (int i = 0; i < dim; ++i) out[i] = (1.0 - t) * v0[i] + t * v1[i];
        return true;
    }
    const double a = sin((1.0 - t) * theta) / st, b = sin(t * theta) / st;
    for (int i = 0; i < dim; ++i) out[i] = a * v0[i] + b * v1[i];
    return true;
}

}  // namespace

int b200_interpolate_vectors(const double* vecs, const double* weights, int n, int dim, int method, double* out,
                             int* out_error_kind) {
    return mb::guarded([&] {
        MB_CHECK_ARG(out_error_kind != nullptr, "out_error_kind is NULL");
        *out_error_kind = B200_INTERP_OK;
        MB_CHECK_ARG(vecs && weights && out, "NULL argument");
        MB_CHECK_ARG(n > 0 && dim > 0, "Cannot interpolate an empty list of vectors");
        MB_CHECK_ARG(method >= B200_INTERP_LERP && method <= B200_INTERP_SLERP, "unknown interpolation method %d", method);
        if (method == B200_INTERP_LERP || method == B200_INTERP_NLERP) {
            double wsum = 0.0;
            for (int i = 0; i < n; ++i) wsum += weights[i];
            if (wsum == 0.0) {
                *out_error_kind = B200_INTERP_ZERO_SUM_WEIGHTS;
                mb::fail(B200_ERR_INVALID_ARG,
                         "Sum of weights is zero. LERP cannot interpolate vectors with zero sum of weights");
            }
            for (int d = 0; d < dim; ++d) out[d] = 0.0;
            for (int i = 0; i < n; ++i) {
                const double w = weights[i] / wsum;
                for (int d = 0; d < dim; ++d) out[d] += w * vecs[(size_t)i * dim + d];
            }
            if (method == B200_INTERP_NLERP) {
                double ss = 0.0;
                for (int d = 0; d < dim; ++d) ss += out[d] * out[d];
                const double len = sqrt(ss);
                if (len == 0.0) {
                    *out_error_kind = B200_INTERP_ZERO_MAGNITUDE;
                    mb::fail(B200_ERR_INVALID_ARG,
                             "Interpolated vector has zero magnitude. Cannot normalize a vector with zero magnitude");
                }
                for (int d = 0; d < dim; ++d) out[d] /= len;
            }
            return;
        }
        // SLERP, hierarchical (the only variant from_interpolation_method builds, :39-40,124-125): neighbours are
        // merged pairwise with t = w1 / (w0 + w1), the merged vector carries weight (w0 + w1) / 2, an odd tail is
        // carried to the next level unchanged (:212-237).
        std::vector<double> cur(vecs, vecs + (size_t)n * dim), next;
        std::vector<double> w(weights, weights + n), nw;
        int m = n;
        while (m > 1) {
            const int half = (m + 1) / 2;
            next.assign((size_t)half * dim, 0.0);
            nw.assign(half, 0.0);
            for (int i = 0; i < m; i += 2) {
                if (i + 1 == m) {
                    std::copy(cur.begin() + (size_t)i * dim, cur.begin() + (size_t)(i + 1) * dim,
                              next.begin() + (size_t)(i / 2) * dim);
                    nw[i / 2] = w[i];
                    continue;
                }
                const double sum = w[i] + w[i + 1];
                if (sum == 0.0) {
                    *out_error_kind = B200_INTERP_ZERO_SUM_WEIGHTS;
                    mb::fail(B200_ERR_INVALID_ARG,
                             "Sum of weights %g and %g is zero. SLERP cannot interpolate vectors with a sum weight of zero",
                             w[i], w[i + 1]);
                }
                if (!slerp_pair(&cur[(size_t)i * dim], &cur[(size_t)(i + 1) * dim], w[i + 1] / sum, dim,
                                &next[(size_t)(i / 2) * dim])) {
                    *out_error_kind = B200_INTERP_ZERO_LENGTH;
                    mb::fail(B200_ERR_INVALID_ARG,
                             "One or more vectors had zero length. SLERP cannot interpolate vectors with zero length");
                }
                nw[i / 2] = sum / 2.0;
            }
            cur.swap(next);
            w.swap(nw);
            m = half;
        }
        std::copy(cur.begin(), cur.begin() + dim, out);
    });
}

}  // extern "C"
