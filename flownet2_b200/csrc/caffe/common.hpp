// Host-side common definitions of the Caffe-surface engine (reference: include/caffe/common.hpp).
// Errors are C++ exceptions (caught at the C-ABI and turned into fn2_status codes) instead of the
// reference's glog CHECK aborts (device_alternate.hpp:48-76).
#pragma once
#include <cuda_runtime.h>

#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../../include/fn2.h"

namespace caffe {

using std::shared_ptr;
using std::string;
using std::vector;

enum Phase { TRAIN = 0, TEST = 1 };

struct CaffeError : std::runtime_error {
    explicit CaffeError(const std::string& m) : std::runtime_error(m) {}
};

struct CheckFail {
    std::ostringstream os;
    CheckFail(const char* file, int line, const char* cond) { os << file << ":" << line << " Check failed: " << cond << " "; }
    template <typename T> CheckFail& operator<<(const T& v) { os << v; return *this; }
    [[noreturn]] ~CheckFail() noexcept(false) { throw CaffeError(os.str()); }
};
#define CHECK(cond) if (cond) {} else ::caffe::CheckFail(__FILE__, __LINE__, #cond)
#define CHECK_EQ(a, b) CHECK((a) == (b)) << "(" << (a) << " vs " << (b) << ") "
#define CHECK_GE(a, b) CHECK((a) >= (b)) << "(" << (a) << " vs " << (b) << ") "
#define CHECK_LE(a, b) CHECK((a) <= (b)) << "(" << (a) << " vs " << (b) << ") "
#define CHECK_GT(a, b) CHECK((a) > (b)) << "(" << (a) << " vs " << (b) << ") "
#define NOT_IMPLEMENTED CHECK(false) << "Not Implemented Yet"

#define CUDA_CHECK(call)                                                              \
    do {                                                                              \
        cudaError_t e__ = (call);                                                     \
        CHECK(e__ == cudaSuccess) << #call << ": " << cudaGetErrorString(e__);         \
    } while (0)

// fn2_* C-ABI call -> exception on failure
#define FN2_CALL(call)                                                                \
    do {                                                                              \
        int rc__ = (call);                                                            \
        CHECK(rc__ == 0) << #call << " -> " << rc__ << ": " << fn2_last_error();       \
    } while (0)

// The reference's Caffe singleton carries mode/device/RNG (common.hpp:100-170); here the only
// thread-local state is the stream layers enqueue on (set by Net around Forward) and the seed.
class Caffe {
 public:
    static cudaStream_t& stream() { static thread_local cudaStream_t s = 0; return s; }
    static uint64_t& seed() { static thread_local uint64_t s = 1701; return s; }
};

// The one owner of host-side CUDA allocations: a cudaMalloc block (or a pinned cudaMallocHost block), freed with the
// object.  reserve() only grows, and frees the old block before it allocates the new one, so peak memory never holds both;
// a failed allocation leaves the buffer empty.  Every allocation is counted process-wide (fn2_device_allocations).
class DeviceBuffer {
 public:
    enum Memory { DEVICE, PINNED_HOST };
    explicit DeviceBuffer(Memory m = DEVICE) : pinned_(m == PINNED_HOST) {}
    ~DeviceBuffer() { release(); }
    DeviceBuffer(DeviceBuffer&& o) noexcept : p_(o.p_), bytes_(o.bytes_), pinned_(o.pinned_) { o.p_ = nullptr; o.bytes_ = 0; }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;

    void reserve(size_t bytes);
    void reserve(size_t bytes, cudaStream_t zero_on);   // a new block is cleared on `zero_on`, which is then synchronised
    void release() noexcept;
    void* get() const { return p_; }
    template <typename T> T* as() const { return static_cast<T*>(p_); }
    size_t bytes() const { return bytes_; }
    bool empty() const { return p_ == nullptr; }

 private:
    void* p_ = nullptr;
    size_t bytes_ = 0;
    bool pinned_;
};

// Dense NCHW view of n x c x h x w floats at p
inline fn2_tensor nchw_view(float* p, int n, int c, int h, int w) {
    fn2_tensor t;
    t.data = p; t.n = n; t.c = c; t.h = h; t.w = w;
    t.sw = 1; t.sh = w; t.sc = (int64_t)h * w; t.sn = (int64_t)c * h * w;
    return t;
}

// Dense NHWC view of n x c x h x w floats at p (channels fastest)
inline fn2_tensor nhwc_view(float* p, int n, int c, int h, int w) {
    fn2_tensor t;
    t.data = p; t.n = n; t.c = c; t.h = h; t.w = w;
    t.sc = 1; t.sw = c; t.sh = (int64_t)w * c; t.sn = (int64_t)h * w * c;
    return t;
}

}  // namespace caffe
