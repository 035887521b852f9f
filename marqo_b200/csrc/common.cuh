// Helpers shared by every translation unit of libmarqo_b200.so:
// status codes, thread-local error text, CUDA error checks, owners of device memory and CUDA handles,
// TMA tensor-map encoding, and the bf16x2 pack of the kernels.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <memory>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>

#include "../../include/marqo_b200.h"

namespace mb {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

void set_last_error(const std::string& msg);

[[noreturn]] inline void fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    throw Error(code, buf);
}

#define MB_CUDA(expr)                                                                                          \
    do {                                                                                                       \
        cudaError_t _e = (expr);                                                                               \
        if (_e != cudaSuccess)                                                                                 \
            ::mb::fail(B200_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

#define MB_CHECK_ARG(cond, ...)                                   \
    do {                                                          \
        if (!(cond)) ::mb::fail(B200_ERR_INVALID_ARG, __VA_ARGS__); \
    } while (0)

// Wraps a C-ABI body: exceptions -> status code + thread-local message.
template <class F>
int guarded(F&& f) {
    try {
        f();
        return B200_OK;
    } catch (const Error& e) {
        set_last_error(e.what());
        return e.code;
    } catch (const std::exception& e) {
        set_last_error(e.what());
        return B200_ERR_INTERNAL;
    }
}

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        MB_CUDA(cudaGetDevice(&prev));
        if (prev != dev) MB_CUDA(cudaSetDevice(dev));
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// Raises B200_ERR_NO_DEVICE / B200_ERR_INVALID_ARG unless `device` is an sm_90 device of this process.
void require_sm90_device(int device);

// ---------------------------------------------------------------------------------------------------- ownership
// Every device allocation of the library goes through device_alloc / device_free: out of memory is reported as
// B200_ERR_OOM, and the process-wide count of live bytes (b200_debug_device_bytes) stays exact.  `stream_ordered`
// selects cudaMallocAsync / cudaFreeAsync on `stream`.
void* device_alloc(size_t bytes, cudaStream_t stream, bool stream_ordered);
void device_free(void* p, size_t bytes, cudaStream_t stream, bool stream_ordered) noexcept;

// Move-only owner of a device array of size() elements.  Default-constructed, moved-from and zero-sized buffers are
// empty (null).
template <class T>
class DeviceBuffer {
  public:
    DeviceBuffer() = default;
    explicit DeviceBuffer(size_t n) : p_(static_cast<T*>(device_alloc(n * sizeof(T), nullptr, false))), n_(n) {}
    // stream-ordered: allocated and released on `s`
    DeviceBuffer(size_t n, cudaStream_t s)
        : p_(static_cast<T*>(device_alloc(n * sizeof(T), s, true))), n_(n), stream_(s), stream_ordered_(true) {}
    DeviceBuffer(DeviceBuffer&& o) noexcept { swap(o); }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
        DeviceBuffer(std::move(o)).swap(*this);
        return *this;
    }
    ~DeviceBuffer() {
        if (p_) device_free(p_, n_ * sizeof(T), stream_, stream_ordered_);
    }
    T* get() const { return p_; }
    size_t size() const { return n_; }
    explicit operator bool() const { return p_ != nullptr; }
    void swap(DeviceBuffer& o) noexcept {
        std::swap(p_, o.p_);
        std::swap(n_, o.n_);
        std::swap(stream_, o.stream_);
        std::swap(stream_ordered_, o.stream_ordered_);
    }

  private:
    T* p_ = nullptr;
    size_t n_ = 0;
    cudaStream_t stream_ = nullptr;
    bool stream_ordered_ = false;
};

struct StreamDeleter {
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};
struct EventDeleter {
    void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
struct GraphExecDeleter {
    void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); }
};
struct PinnedDeleter {
    void operator()(void* p) const { cudaFreeHost(p); }
};
struct IpcDeleter {
    void operator()(void* p) const { cudaIpcCloseMemHandle(p); }
};
using UniqueStream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDeleter>;
using UniqueEvent = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDeleter>;
using UniqueGraphExec = std::unique_ptr<std::remove_pointer_t<cudaGraphExec_t>, GraphExecDeleter>;
template <class T>
using PinnedPtr = std::unique_ptr<T, PinnedDeleter>;
using IpcMapping = std::unique_ptr<uint8_t, IpcDeleter>;   // another process's device buffer mapped here

UniqueStream make_stream(unsigned flags);
UniqueEvent make_event();
void* pinned_alloc(size_t bytes);   // portable page-locked host memory
template <class T>
PinnedPtr<T> make_pinned() {
    return PinnedPtr<T>(static_cast<T*>(pinned_alloc(sizeof(T))));
}
IpcMapping open_ipc_mapping(const cudaIpcMemHandle_t& h);

// 2D row-major tensor map: inner dim `cols` (contiguous), outer dim `rows`, row pitch in bytes.
// box = {box_cols, box_rows}; swizzle 128B requires box_cols * elem_size == 128.
CUtensorMap make_tmap_2d(const void* base, CUtensorMapDataType dtype, uint32_t elem_bytes, uint64_t cols,
                         uint64_t rows, uint64_t row_pitch_bytes, uint32_t box_cols, uint32_t box_rows,
                         CUtensorMapSwizzle swizzle);

int sm_count(int device);

inline size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// (lo, hi) rounded to bf16 (round to nearest even) in one 32-bit word, lo in the low half
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}

}  // namespace mb
