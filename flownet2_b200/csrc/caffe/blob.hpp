// Blob: the tensor type of the Caffe layer surface (reference: include/caffe/blob.hpp:23-280,
// src/caffe/syncedmem.cpp).  Logical shape and host view are NCHW exactly like the reference
// (offset = ((n*C+c)*H+h)*W+w, blob.hpp:153-163).  Device storage is fp32 in one of two layouts:
//   PLAIN : dense NCHW (parameters; what a reference layer's gpu_data() would see)
//   NHWC  : channel-fastest with a padded pixel stride (activations inside the engine; the
//           the tensor-core conv wants K-major operands and Correlation/FlowWarp want per-pixel vectors;
//           the reference converts to NHWC inside those two layers anyway,
//           correlation_layer.cu:41, flow_warp_layer.cu:51)
// cpu_data()/mutable_cpu_data() keep the reference's lazy host<->device mirroring semantics.
#pragma once
#include "common.hpp"
#include "proto.hpp"

namespace caffe {

template <typename Dtype>
class Blob {
 public:
    enum Layout { PLAIN = 0, NHWC = 1 };
    Blob() {}
    explicit Blob(int n, int c, int h, int w) { Reshape(n, c, h, w); }
    Blob(const Blob&) = delete;
    Blob& operator=(const Blob&) = delete;

    void Reshape(int n, int c, int h, int w);
    void Reshape(const vector<int>& shape);
    void ReshapeLike(const Blob& o) { Reshape(o.shape_); }
    // Layout of the device storage; must be chosen before the first device access.
    // channel_align < 0: automatic (4 below 32 channels, else 32 -- the tensor-core conv K block)
    void set_layout(Layout l, int channel_align = -1);
    Layout layout() const { return layout_; }

    const vector<int>& shape() const { return shape_; }
    int num_axes() const { return (int)shape_.size(); }
    int shape(int i) const { return i < (int)shape_.size() ? shape_[i] : 1; }
    int num() const { return shape(0); }
    int channels() const { return shape(1); }
    int height() const { return shape(2); }
    int width() const { return shape(3); }
    int count() const { return count_; }
    int offset(int n, int c = 0, int h = 0, int w = 0) const { return ((n * channels() + c) * height() + h) * width() + w; }

    // Host view (NCHW).  Syncs from the device if the device copy is newer.
    const Dtype* cpu_data();
    Dtype* mutable_cpu_data();
    // Raw device storage in layout().  PLAIN blobs: exactly the reference's gpu_data().
    const Dtype* gpu_data();
    Dtype* mutable_gpu_data();
    // Strided view for the fn2_* C-ABI; channel sub-range [c0, c0+cn) (cn<0: to the end).
    fn2_tensor tensor(int c0 = 0, int cn = -1);
    fn2_tensor mutable_tensor(int c0 = 0, int cn = -1);
    // Gradient storage (blob.hpp:230-246 cpu_diff / gpu_diff): same device layout as the data, allocated on first use.  A
    // zero-copy concat child's diff is the matching channel range of its parent's diff.
    fn2_tensor diff_tensor(int c0 = 0, int cn = -1);
    const Dtype* cpu_diff();                  // NCHW host copy of the gradient (downloads)
    void set_cpu_diff(const Dtype* host_nchw);  // uploads
    void ZeroDiff(cudaStream_t st);
    bool has_diff() const { return ddev_ != nullptr || (parent_ && parent_->has_diff()); }
    size_t storage_floats() const;            // device floats incl. channel padding
    int channel_stride() const { return cstride_; }

    // Make this blob a channel-range view [c0, c0+channels) into `parent`'s NHWC storage
    // (zero-copy Concat).  The blob keeps its own logical shape.
    static constexpr int kGuardFloats = 256;   // guard band (floats) before and after every owned device allocation
    void AliasInto(Blob* parent, int c0);
    bool is_alias() const { return parent_ != nullptr; }
    const Blob* alias_parent() const { return parent_; }
    int alias_offset() const { return parent_c0_; }
    // Bind PLAIN storage to external device memory (the Net's parameter arena); current contents
    // are copied there.
    void BindExternal(Dtype* dev);
    void BindExternalDiff(Dtype* dev);         // gradient arena (contiguous parameter diffs: one all-reduce for data parallelism)
    void ShareData(Blob& other);
    // The device copy was written behind the blob's back (arena broadcast, CUDA-graph replay): the next cpu_data() must
    // download it again instead of trusting the cached host copy.
    void MarkDeviceNewer();

    void FromProto(const BlobProtoData& p, bool reshape = true);   // blob.cpp:436-490
    void ToProto(BlobProtoData* p);

 private:
    void alloc_device();
    void to_cpu();
    void to_gpu();
    enum Head { UNINIT, AT_CPU, AT_GPU, SYNCED };
    vector<int> shape_;
    int count_ = 0;
    Layout layout_ = PLAIN;
    int calign_ = -1;
    int compute_cstride() const;
    int cstride_ = 0;             // pixel stride (floats) for NHWC
    Head head_ = UNINIT;
    vector<Dtype> host_;
    // dev_ / ddev_ point kGuardFloats into data_ / diff_ while those own the storage (non-empty); aliased, arena-bound and
    // shared storage is a plain pointer with the buffer empty
    Dtype* dev_ = nullptr;
    DeviceBuffer data_;
    Dtype* ddev_ = nullptr;       // gradient storage
    DeviceBuffer diff_;
    vector<Dtype> dhost_;
    Blob* parent_ = nullptr;      // alias target
    int parent_c0_ = 0;
};

}  // namespace caffe
