// input_stager.hpp -- the input path of train(), train_accumulate() and train_raw() (DESIGN.md row f3).
//
// The reference keeps a 2-deep Free/Full queue of host blobs between the transformer threads and the solver thread
// (CaffeProcessor.scala:32-35,442-452) and MemoryInputAdapter::feed points the data layer at the host blob
// (MemoryInputAdapter.cpp:24-32).  Here: two device-side staging sets; the H2D copy of batch t runs on its own copy
// stream while the compute stream still works on batch t-1; train() returns as soon as ITS batch has left host memory
// (the caller recycles the blobs after train() returns).
#ifndef COS_INPUT_STAGER_HPP_
#define COS_INPUT_STAGER_HPP_

#include <cuda_runtime_api.h>

#include <memory>
#include <string>
#include <vector>

#include "../../include/caffedistri_b200.h"
#include "data_transform.hpp"
#include "solver_spec.hpp"

namespace cosb {

// A buffer that frees itself and never shrinks: device memory, or pinned host memory when Pinned.
template <bool Pinned>
class GrowBuffer {
 public:
  void* get() const { return p_.get(); }
  // At least n bytes.  A smaller buffer is freed once `stream`, which may still read it, has finished.
  cudaError_t grow(size_t n, cudaStream_t stream) {
    if (n == 0 || (p_ && n <= bytes_)) return cudaSuccess;
    cudaError_t e = p_ ? cudaStreamSynchronize(stream) : cudaSuccess;
    if (e != cudaSuccess) return e;
    p_.reset();
    void* p = nullptr;
    e = Pinned ? cudaMallocHost(&p, n) : cudaMalloc(&p, n);
    if (e == cudaSuccess) p_.reset(p);
    bytes_ = n;
    return e;
  }

 private:
  struct Free {
    void operator()(void* p) const { Pinned ? cudaFreeHost(p) : cudaFree(p); }
  };
  std::unique_ptr<void, Free> p_;
  size_t bytes_ = 0;  // of p_, when there is one
};
using DeviceBuffer = GrowBuffer<false>;
using PinnedBuffer = GrowBuffer<true>;

class InputStager {
 public:
  // The copy stream and the stages' events on `device`; `compute` is the stream the producer runs on.
  bool create(int device, cudaStream_t compute, std::string* err);
  // Frees every buffer, event and the copy stream.  The device must be idle.
  void release();
  // train_raw's argument checks.  The first call that passes resolves the transforms, uploads their means and keeps
  // its raw shapes, which every later call must repeat; a refused call changes nothing.
  bool check_raw(const SolverSpec& spec, const cos_raw_blob* data, int ndata, std::string* err);
  // Queues this step's nblobs host blobs (from `raw` for train_raw, else `data`) on the copy stream into the current
  // stage and makes the compute stream wait for them.  *in gets the fp32 blobs the producer reads.
  bool stage(const cos_blob* data, const cos_raw_blob* raw, int nblobs, std::vector<cos_blob>* in, std::string* err);
  // Pass `pass` of a train_raw step on the compute stream: every input with a transform_param, from the stage's raw
  // set into its fp32 set.
  bool transform(int64_t seed, int rank, int iter, int pass, std::string* err);
  // The compute stream is done with the stage once it gets here; the next step stages into the other one.
  bool mark_consumed(std::string* err);
  // Waits until the last staged step's host blobs have been read.
  bool wait_copied(std::string* err);

 private:
  struct Input {
    DeviceBuffer fp32;      // what the producer reads
    DeviceBuffer raw;       // train_raw: the untransformed input when it has a transform_param
                            // (COS_RAW_U8_IMAGES: a ragged arena, grown to the largest batch seen)
    DeviceBuffer geom;      // COS_RAW_U8_IMAGES: the call's ImageGeometry table on the device
    PinnedBuffer geom_host;  // ... and in pinned host memory, the source of its copy
  };
  struct Stage {
    std::vector<Input> inputs;
    cudaEvent_t copied = nullptr;    // H2D of this stage finished
    cudaEvent_t consumed = nullptr;  // the step that read this stage finished
    bool consumed_valid = false;
  };
  int device_ = -1;
  cudaStream_t compute_ = nullptr;
  cudaStream_t copy_ = nullptr;
  Stage stages_[2];
  int idx_ = 0;
  // train_raw: the staged inputs' transforms with their means on this device, and the first call's raw shapes
  std::vector<InputTransform> transforms_;
  std::vector<DeviceBuffer> means_;
  std::vector<cos_raw_blob> raw_shapes_;
};

}  // namespace cosb
#endif
