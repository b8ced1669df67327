// native_producer.hpp -- the built-in gradient producer (Net::ForwardBackward for the TRAIN phase of the LeNet,
// CIFAR-10-quick, CIFAR-10-full, CIFAR-10-full-BN and siamese MNIST family of nets, least-squares regression nets and
// residual nets built of Split, Eltwise and Scale; DESIGN.md section 14).
//
// build_plan() turns the layout parser's TRAIN-phase layer list (solver_spec.hpp: the shape inference is shared
// with the learnable layout) into an ordered op list with shapes, in-place aliasing and the flat data_/diff_ offset
// of every learnable blob, or refuses the net naming the first layer it cannot run.  NativeProducer holds the device
// buffers of one plan on one device and enqueues forward + backward (native_producer.cu).
#ifndef COS_NATIVE_PRODUCER_HPP_
#define COS_NATIVE_PRODUCER_HPP_

#include <cuda_runtime_api.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/caffedistri_b200.h"
#include "solver_spec.hpp"

namespace cosb {

enum class OpKind {
  kConv, kConvBiasReluMaxPool, kPool, kInnerProduct, kReLU, kSigmoid, kBatchNorm, kSoftmaxLoss, kLRNWithin, kSlice,
  kContrastiveLoss, kConcat, kEuclideanLoss, kSplit, kEltwise, kScale,
  kCount  // the number of kinds (Plan::text names each)
};

enum EltwiseOp { kEltwiseProd = 0, kEltwiseSum = 1, kEltwiseMax = 2 };  // caffe.proto EltwiseParameter numbering

struct Op {
  OpKind kind;
  std::string name;                    // layer name (the fused block: "conv1+relu1+pool1")
  // tensor ids of the bottoms, in the layer's bottom order, and whether each gets a data gradient: not a staged input,
  // nor a blob that no learnable blob precedes (Caffe's bottom_need_backward), nor the label-like bottom.
  // SoftmaxWithLoss writes its bottom's gradient whatever the flag says.
  std::vector<int> bottoms;
  std::vector<bool> bottom_grad;
  // the label-like bottom (SoftmaxWithLoss's label, ContrastiveLoss's sim), or -1: read, never differentiated, and not
  // counted as its blob's reader
  int label_bottom = -1;
  int out = -1;                        // tensor id of the top
  std::vector<int64_t> in_shape, out_shape;  // in_shape: bottoms[0]'s
  bool in_place = false;               // ReLU / Sigmoid with top == bottom: out shares bottoms[0]'s storage (never a
                                       // staged input's: those are not written)
  // Convolution, Pooling, the fused block's convolution
  int kh = 0, kw = 0, sh = 1, sw = 1, ph = 0, pw = 0;
  bool max_pool = true;
  int pool_kernel = 0, pool_stride = 0;  // the fused block's MAX pool (square, pad 0)
  int64_t w_off = -1, w_count = 0, b_off = -1, b_count = 0;  // flat offsets into data_ / diff_
  std::vector<int> shares;             // learnable blobs this op uses as a sharer of a named param (owned elsewhere)
  float slope = 0.f;                   // ReLU negative_slope
  float loss_weight = 1.f;             // SoftmaxWithLoss, ContrastiveLoss, EuclideanLoss
  bool global_stats = false;           // BatchNorm
  float fraction = 0.999f, eps = 1e-5f;
  int lrn_size = 0;                    // LRN (WITHIN_CHANNEL only)
  float lrn_alpha = 1.f, lrn_beta = 0.75f;
  // Slice: this op copies bottom[.., slice_begin .. slice_begin + out_shape[slice_axis], ..] to its one top.
  // Concat, the inverse: this op copies its one bottom to top[.., slice_begin .. slice_begin + in_shape[slice_axis], ..]
  int slice_axis = 0;
  int64_t slice_begin = 0;
  float margin = 1.f;                  // ContrastiveLoss
  bool legacy = false;
  // Split: this op's top index.  Its top's activation is the bottom's (Plan::data_alias); the op of top 0 sums the
  // gradients of split_sum (the tops some layer reads, in top order) into the bottom's, and the others do nothing.
  int split_top = 0;
  std::vector<int> split_sum;
  bool split_unread = false;           // no layer reads this top: it adds nothing to the bottom's gradient
  // Eltwise: coeffs for SUM, one per bottom
  int eltwise_op = kEltwiseSum;
  std::vector<float> coeffs;
  bool stable_prod_grad = true;
  // Scale: y[o, d, i] = x[o, d, i] * s[d] (+ b[d]) over outer o, scale_dim d and inner i; w_off / b_off are s and b
  int64_t scale_outer = 1, scale_dim = 1, scale_inner = 1;
};

struct Plan {
  std::vector<Op> ops;
  std::vector<int64_t> tensor_count;   // elements per tensor id
  std::vector<int> storage;            // tensor id -> tensor id that owns its memory (itself unless in place)
  // per tensor id: its activation is another tensor's memory, set when the forward reaches it (a Split top reads its
  // bottom's, as Caffe's ShareData); its gradient is still its own
  std::vector<bool> data_alias;
  int ninputs = 0;                     // tensors 0 .. ninputs-1 are the staged inputs, in data-layer top order
  std::vector<std::string> input_names;
  std::vector<int64_t> blob_off, blob_count;  // every learnable blob, learnable_params() order
  std::vector<std::vector<int64_t>> blob_shape;
  std::vector<FillerSpec> blob_filler;
  int64_t param_count = 0;
  std::string text() const;  // one op per line (cos_native_producer_plan)
};

// Builds the plan of a parsed TRAIN net (a Slice or Split layer becomes one op per top, a Concat layer one kConcat op
// per bottom, each with one bottom); false with "layer '<name>' (<type>): <reason>" when it cannot be run.
bool build_plan(const SolverSpec& spec, const std::vector<NetLayer>& layers, Plan* plan, std::string* err);
// parse_train_net + build_plan.
bool plan_from_prototxt(const std::string& path, SolverSpec* spec, Plan* plan, std::string* err);

// Status word value of a label outside [0, classes) (CaffeNet::check_status turns it into an error).
constexpr int kStatusBadLabel = 500;

class NativeProducer {
 public:
  // Allocates every activation, gradient, index, BatchNorm save area and split-K workspace of `plan` on `device`.
  static NativeProducer* create(const Plan& plan, int device, float* data, float* diff, int* status, std::string* err);
  ~NativeProducer();
  // Fills data_ from the prototxt fillers with the counter-based generator keyed by (seed, blob index).  Synchronous.
  bool fill(uint64_t seed, cudaStream_t stream, std::string* err);
  // One forward + backward on `stream`: accumulates every gradient into diff_ once and writes the loss.  Only enqueues
  // (no allocation, synchronisation or device query).  0 on success, else a cudaError_t or -1 for bad inputs.
  int forward_backward(const cos_blob* inputs, int ninputs, float* loss_dev, cudaStream_t stream);
  // cos_forward_backward_fn trampoline; `user` is the NativeProducer
  static int callback(void* user, int solver_index, const cos_blob* inputs, int ninputs, float* loss_dev,
                      void* cuda_stream);

 private:
  NativeProducer(const Plan& plan, int device, float* data, float* diff, int* status)
      : plan_(plan), device_(device), data_(data), diff_(diff), status_(status) {}
  bool allocate(std::string* err);
  cudaError_t run_op_forward(const Op& op, size_t i, float* loss_dev, cudaStream_t s);
  cudaError_t run_op_backward(const Op& op, size_t i, cudaStream_t s);

  Plan plan_;
  int device_;
  float* data_;
  float* diff_;
  int* status_;
  std::vector<float*> act_, grad_;        // per tensor id (staged inputs: act_ is the caller's buffer, set per call)
  std::vector<void*> op_aux_;             // per op: MAX pool / Eltwise MAX argmax (int32), fused block index (uint8),
                                          // BN save
  std::vector<float*> op_z_, op_dz_;      // fused block: conv output without bias and its gradient
  cudaEvent_t done_ = nullptr;            // recorded at the end of every call: the destructor waits for it
  float* workspace_ = nullptr;            // split-K partials, bias partials, BatchNorm scratch (ops run in order)
  size_t workspace_floats_ = 0;
  std::vector<void*> allocations_;
};

}  // namespace cosb
#endif
