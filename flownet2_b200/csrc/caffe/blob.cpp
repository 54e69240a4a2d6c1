#include "blob.hpp"

#include <algorithm>
#include <atomic>
#include <cstring>

namespace caffe {

// ---- DeviceBuffer -----------------------------------------------------------------------------------------------------
static std::atomic<uint64_t> g_allocations{0}, g_live_bytes{0};

DeviceBuffer& DeviceBuffer::operator=(DeviceBuffer&& o) noexcept {
    if (this != &o) {
        release();
        p_ = o.p_; bytes_ = o.bytes_; pinned_ = o.pinned_;
        o.p_ = nullptr; o.bytes_ = 0;
    }
    return *this;
}

void DeviceBuffer::release() noexcept {
    if (!p_) return;
    if (pinned_) cudaFreeHost(p_);
    else cudaFree(p_);
    g_live_bytes -= bytes_;
    p_ = nullptr; bytes_ = 0;
}

void DeviceBuffer::reserve(size_t bytes) {
    if (bytes <= bytes_) return;
    release();
    void* p = nullptr;
    const cudaError_t e = pinned_ ? cudaMallocHost(&p, bytes) : cudaMalloc(&p, bytes);
    CHECK(e == cudaSuccess) << (pinned_ ? "cudaMallocHost" : "cudaMalloc") << " of " << bytes << " bytes: " << cudaGetErrorString(e);
    p_ = p; bytes_ = bytes;
    g_allocations++; g_live_bytes += bytes;
}

void DeviceBuffer::reserve(size_t bytes, cudaStream_t zero_on) {
    if (bytes <= bytes_) return;
    reserve(bytes);
    CUDA_CHECK(cudaMemsetAsync(p_, 0, bytes, zero_on));
    CUDA_CHECK(cudaStreamSynchronize(zero_on));
}

// Copies between a device view and a dense host NCHW array through a dense device temporary (fn2_copy changes the layout).
static void copy_nchw(const fn2_tensor& view, float* host, cudaMemcpyKind dir, cudaStream_t st) {
    const size_t bytes = (size_t)view.n * view.c * view.h * view.w * sizeof(float);
    DeviceBuffer tmp;
    tmp.reserve(bytes);
    const fn2_tensor dense = nchw_view(tmp.as<float>(), view.n, view.c, view.h, view.w);
    if (dir == cudaMemcpyDeviceToHost) {
        FN2_CALL(fn2_copy(&view, &dense, st));
        CUDA_CHECK(cudaMemcpyAsync(host, tmp.get(), bytes, dir, st));
    } else {
        CUDA_CHECK(cudaMemcpyAsync(tmp.get(), host, bytes, dir, st));
        FN2_CALL(fn2_copy(&dense, &view, st));
    }
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// ---- gradient storage -------------------------------------------------------------------------------------------------
template <typename Dtype>
fn2_tensor Blob<Dtype>::diff_tensor(int c0, int cn) {
    if (parent_) {
        fn2_tensor pt = parent_->diff_tensor(parent_c0_ + c0, cn < 0 ? channels() - c0 : cn);
        return pt;
    }
    if (!ddev_ || !diff_.empty()) {                           // owned storage grows with the blob
        ddev_ = nullptr;
        diff_.reserve((std::max<size_t>(storage_floats(), 1) + 2 * kGuardFloats) * sizeof(Dtype), Caffe::stream());
        ddev_ = diff_.as<Dtype>() + kGuardFloats;
    }
    mutable_gpu_data();                                       // make sure the data view (strides) exists
    Head h = head_;
    fn2_tensor t = mutable_tensor(c0, cn);
    head_ = h;
    t.data = ddev_ + (t.data - dev_);
    return t;
}

template <typename Dtype>
void Blob<Dtype>::BindExternalDiff(Dtype* dev) {
    CHECK(layout_ == PLAIN && !parent_) << "only PLAIN blobs can be bound to the gradient arena";
    diff_.release();
    ddev_ = dev;
}

template <typename Dtype>
void Blob<Dtype>::ZeroDiff(cudaStream_t st) {
    if (parent_) return;                                      // cleared with the parent
    if (!ddev_) { diff_tensor(); return; }                    // fresh allocation is already zero
    CUDA_CHECK(cudaMemsetAsync(ddev_, 0, storage_floats() * sizeof(Dtype), st));
}

template <typename Dtype>
const Dtype* Blob<Dtype>::cpu_diff() {
    dhost_.resize((size_t)count_);
    if (count_ == 0) return dhost_.data();
    copy_nchw(diff_tensor(), dhost_.data(), cudaMemcpyDeviceToHost, Caffe::stream());
    return dhost_.data();
}

template <typename Dtype>
void Blob<Dtype>::set_cpu_diff(const Dtype* host_nchw) {
    if (count_ == 0) return;
    copy_nchw(diff_tensor(), const_cast<Dtype*>(host_nchw), cudaMemcpyHostToDevice, Caffe::stream());
}

template <typename Dtype>
void Blob<Dtype>::Reshape(int n, int c, int h, int w) {
    vector<int> s = {n, c, h, w};
    Reshape(s);
}

template <typename Dtype>
void Blob<Dtype>::Reshape(const vector<int>& shape) {
    CHECK_LE(shape.size(), 4u) << "blobs of more than 4 axes are not used on the FlowNet2 path";
    long long cnt = 1;
    for (int d : shape) {
        CHECK_GE(d, 0);
        cnt *= d;
        CHECK_LE(cnt, 2147483647LL) << "blob size exceeds INT_MAX (blob.cpp:33)";
    }
    if (shape == shape_ && count_ == (int)cnt) return;
    CHECK(!parent_) << "cannot reshape an aliased blob";
    // externally bound storage (a slot of the Net's parameter arena, or another blob's buffer) has a fixed size
    CHECK(!data_.empty() || !dev_ || (long long)count_ == cnt)
        << "cannot reshape a blob bound to external storage to a different count (" << count_ << " -> " << cnt << ")";
    shape_ = shape;
    count_ = (int)cnt;
    cstride_ = compute_cstride();
    if (!data_.empty()) { data_.release(); dev_ = nullptr; }
    host_.clear();
    head_ = UNINIT;
}

template <typename Dtype>
void Blob<Dtype>::set_layout(Layout l, int channel_align) {
    CHECK(!dev_ || (l == layout_ && channel_align == calign_)) << "layout must be set before device allocation";
    layout_ = l;
    calign_ = channel_align;
    cstride_ = compute_cstride();
}

template <typename Dtype>
int Blob<Dtype>::compute_cstride() const {
    if (layout_ != NHWC) return 0;
    const int c = channels();
    const int a = calign_ > 0 ? calign_ : (c < 32 ? 4 : 32);
    return (c + a - 1) / a * a;
}

template <typename Dtype>
size_t Blob<Dtype>::storage_floats() const {
    if (layout_ == PLAIN) return (size_t)count_;
    return (size_t)num() * height() * width() * cstride_;
}

template <typename Dtype>
void Blob<Dtype>::alloc_device() {
    if (parent_) {
        parent_->mutable_gpu_data();
        dev_ = parent_->dev_ + parent_c0_;
        return;
    }
    if (dev_) return;
    // kGuardFloats readable floats on both sides: the small-Ci tensor-core convolution fetches whole kernel rows and
    // reaches a few pixels outside the tensor at the image corners (those values are masked, never used).
    // Zeroed because channel padding must read as zero forever (weights for padded channels are zero, but 0 * NaN would
    // poison the tensor-core path); stream-ordered, because the nets run on non-blocking streams and a legacy-stream memset
    // could land AFTER the first kernel that writes the blob
    data_.reserve((std::max<size_t>(storage_floats(), 1) + 2 * kGuardFloats) * sizeof(Dtype), Caffe::stream());
    dev_ = data_.as<Dtype>() + kGuardFloats;
}

template <typename Dtype>
fn2_tensor Blob<Dtype>::mutable_tensor(int c0, int cn) {
    Dtype* p = mutable_gpu_data();
    fn2_tensor t;
    if (cn < 0) cn = channels() - c0;
    CHECK(c0 >= 0 && cn > 0 && c0 + cn <= channels()) << "bad channel range";
    t.n = num(); t.c = cn; t.h = height(); t.w = width();
    if (layout_ == PLAIN) {
        t.sw = 1; t.sh = width(); t.sc = (int64_t)height() * width(); t.sn = (int64_t)channels() * height() * width();
        t.data = p + (int64_t)c0 * t.sc;
    } else {
        const int cs = parent_ ? parent_->cstride_ : cstride_;
        t.sc = 1; t.sw = cs; t.sh = (int64_t)width() * cs; t.sn = (int64_t)height() * width() * cs;
        t.data = p + c0;
    }
    return t;
}

template <typename Dtype>
fn2_tensor Blob<Dtype>::tensor(int c0, int cn) {
    gpu_data();
    Head h = head_;
    fn2_tensor t = mutable_tensor(c0, cn);
    head_ = h;
    return t;
}

template <typename Dtype>
void Blob<Dtype>::to_cpu() {
    if (head_ == UNINIT) {
        host_.assign((size_t)count_, Dtype(0));
        head_ = AT_CPU;
        return;
    }
    if (head_ != AT_GPU) return;
    host_.resize((size_t)count_);
    if (count_ == 0) { head_ = SYNCED; return; }
    cudaStream_t st = Caffe::stream();
    if (layout_ == PLAIN && !parent_) {
        CUDA_CHECK(cudaMemcpyAsync(host_.data(), dev_, (size_t)count_ * sizeof(Dtype), cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    } else {
        Head h = head_;
        fn2_tensor src = mutable_tensor();
        head_ = h;
        copy_nchw(src, host_.data(), cudaMemcpyDeviceToHost, st);
    }
    head_ = SYNCED;
}

template <typename Dtype>
void Blob<Dtype>::to_gpu() {
    if (head_ == UNINIT) {
        alloc_device();
        head_ = AT_GPU;
        return;
    }
    if (head_ != AT_CPU) { alloc_device(); return; }
    alloc_device();
    if (count_ == 0) { head_ = SYNCED; return; }
    cudaStream_t st = Caffe::stream();
    if (layout_ == PLAIN && !parent_) {
        CUDA_CHECK(cudaMemcpyAsync(dev_, host_.data(), (size_t)count_ * sizeof(Dtype), cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    } else {
        head_ = SYNCED;
        copy_nchw(mutable_tensor(), host_.data(), cudaMemcpyHostToDevice, st);
    }
    head_ = SYNCED;
}

template <typename Dtype>
const Dtype* Blob<Dtype>::cpu_data() {
    to_cpu();
    return host_.data();
}
template <typename Dtype>
Dtype* Blob<Dtype>::mutable_cpu_data() {
    to_cpu();
    head_ = AT_CPU;
    return host_.data();
}
template <typename Dtype>
const Dtype* Blob<Dtype>::gpu_data() {
    to_gpu();
    return dev_;
}
template <typename Dtype>
Dtype* Blob<Dtype>::mutable_gpu_data() {
    to_gpu();
    head_ = AT_GPU;
    if (parent_) parent_->head_ = AT_GPU;
    return dev_;
}

template <typename Dtype>
void Blob<Dtype>::AliasInto(Blob* parent, int c0) {
    CHECK(parent && parent->layout_ == NHWC && layout_ == NHWC) << "aliasing needs NHWC blobs";
    CHECK(data_.empty() || head_ == UNINIT) << "blob already has device data";
    CHECK(num() == parent->num() && height() == parent->height() && width() == parent->width());
    CHECK(c0 >= 0 && c0 + channels() <= parent->channels());
    data_.release();
    dev_ = nullptr;
    parent_ = parent;
    parent_c0_ = c0;
    cstride_ = parent->cstride_;
}

template <typename Dtype>
void Blob<Dtype>::BindExternal(Dtype* dev) {
    CHECK(layout_ == PLAIN && !parent_) << "only PLAIN blobs can be bound to the parameter arena";
    const Dtype* h = cpu_data();           // bring current contents to the host
    data_.release();
    dev_ = dev;
    if (count_) CUDA_CHECK(cudaMemcpy(dev_, h, (size_t)count_ * sizeof(Dtype), cudaMemcpyHostToDevice));
    head_ = SYNCED;
}

template <typename Dtype>
void Blob<Dtype>::MarkDeviceNewer() {
    if (dev_ || parent_) head_ = AT_GPU;
}

template <typename Dtype>
void Blob<Dtype>::ShareData(Blob& other) {
    CHECK_EQ(count_, other.count_);
    CHECK(layout_ == other.layout_);
    other.gpu_data();
    data_.release();
    dev_ = other.dev_;
    cstride_ = other.cstride_;
    head_ = AT_GPU;
}

template <typename Dtype>
void Blob<Dtype>::FromProto(const BlobProtoData& p, bool reshape) {
    if (reshape) {
        vector<int> s = p.shape;
        CHECK_LE(s.size(), 4u);
        Reshape(s);
    } else {
        // shape must match up to leading 1s like Blob::ShapeEquals (blob.cpp:407-432)
        long long cnt = 1;
        for (int d : p.shape) cnt *= d;
        CHECK_EQ((long long)count_, cnt) << "shape mismatch (reshape not set)";
    }
    CHECK_EQ((size_t)count_, p.data.size()) << "blob data size mismatch";
    Dtype* d = mutable_cpu_data();
    for (int i = 0; i < count_; i++) d[i] = (Dtype)p.data[i];
}

template <typename Dtype>
void Blob<Dtype>::ToProto(BlobProtoData* p) {
    p->shape = shape_;
    const Dtype* d = cpu_data();
    p->data.assign(d, d + count_);
}

template class Blob<float>;

}  // namespace caffe

uint64_t fn2_device_allocations(uint64_t* live_bytes) {
    if (live_bytes) *live_bytes = caffe::g_live_bytes;
    return caffe::g_allocations;
}
