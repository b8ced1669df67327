// native_producer.hpp -- the built-in gradient producer (Net::ForwardBackward for the TRAIN phase of the LeNet,
// CIFAR-10-quick, CIFAR-10-full, CIFAR-10-full-BN and siamese MNIST family of nets, least-squares regression nets,
// residual nets built of Split, Eltwise and Scale, autoencoders built of Flatten, Deconvolution and
// SigmoidCrossEntropyLoss, embedding nets that read token ids through Embed and Reshape, recurrent nets built of
// RNN layers over time-major inputs, and nets normalised by MVN; DESIGN.md section 14).
//
// build_plan() turns the layout parser's TRAIN-phase layer list (solver_spec.hpp: the shape inference is shared
// with the learnable layout) into an ordered op list with shapes, in-place aliasing and the flat data_/diff_ offset
// of every learnable blob, or refuses the net naming the first layer it cannot run.  Only the ops under the loss run a
// backward (Caffe's layer_need_backward): an op whose top no gradient reaches runs its forward alone.  A loss layer
// with loss_weight 0 does no TRAIN work at all.  NativeProducer holds the device
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
  kContrastiveLoss, kConcat, kEuclideanLoss, kSplit, kEltwise, kScale, kDeconv, kFlatten, kSigmoidCrossEntropyLoss,
  kTanH, kELU, kAbsVal, kBNLL, kPower, kExp, kLog, kThreshold, kPReLU, kSoftmax, kMultinomialLogisticLoss, kHingeLoss,
  kEmbed, kReshape, kRNN, kMVN,
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
  // the label-like bottom (SoftmaxWithLoss's label, ContrastiveLoss's sim, SigmoidCrossEntropyLoss's target), or -1:
  // read, never differentiated, and not counted as its blob's reader
  int label_bottom = -1;
  // no gradient reaches the top (it is read by no layer under the loss, or only as a label): the op runs its forward
  // and no backward.  Never set on a Split op (such a top is split_unread) nor a Slice op (it still writes its range of
  // the bottom's gradient).
  bool no_backward = false;
  int out = -1;                        // tensor id of the top
  std::vector<int64_t> in_shape, out_shape;  // in_shape: bottoms[0]'s
  bool in_place = false;               // ReLU / Sigmoid with top == bottom: out shares bottoms[0]'s storage (never a
                                       // staged input's: those are not written)
  // Convolution, Deconvolution, Pooling, the fused block's convolution
  int kh = 0, kw = 0, sh = 1, sw = 1, ph = 0, pw = 0;
  bool max_pool = true;
  int pool_kernel = 0, pool_stride = 0;  // the fused block's MAX pool (square, pad 0)
  int64_t w_off = -1, w_count = 0, b_off = -1, b_count = 0;  // flat offsets into data_ / diff_
  std::vector<int> shares;             // learnable blobs this op uses as a sharer of a named param (owned elsewhere)
  float slope = 0.f;                   // ReLU negative_slope
  float loss_weight = 1.f;             // SoftmaxWithLoss, ContrastiveLoss, EuclideanLoss, SigmoidCrossEntropyLoss
  // SoftmaxWithLoss (softmax_loss_layer.cpp Reshape): the class axis and its C classes; rows = count(0, axis) *
  // inner, one label each, with inner = count(axis + 1)
  int softmax_axis = 1;
  int64_t classes = 0, rows = 0, inner = 1;
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
  // The neuron ops (Caffe's *_layer.cpp LayerSetUp, computed in float as Caffe does): ELU's alpha; Power's power, scale
  // and shift; Exp's inner_scale = log(base) * scale and outer_scale = base^shift; Log's scale, shift, base_scale =
  // 1 / log(base) and backward_num_scale = scale / log(base); Threshold's threshold.  base is kept for the plan line.
  float alpha = 1.f, power = 1.f, scale = 1.f, shift = 0.f, base = -1.f;
  float inner_scale = 1.f, outer_scale = 1.f, base_scale = 1.f, backward_num_scale = 1.f;
  float threshold = 0.f;
  // PReLU: the slope blob is w_off; y[n, c, p] uses slope[channel_shared ? 0 : c] over prelu_channels C and
  // prelu_dim = count(2) elements per (n, c)
  bool channel_shared = false;
  int64_t prelu_channels = 1, prelu_dim = 1;
  // Softmax: softmax_axis, classes and inner as SoftmaxWithLoss's, outer = count(0, axis)
  int64_t outer = 1;
  bool hinge_l2 = false;               // HingeLoss: L2 norm (else L1)
  // Embed: the vocabulary size K (w_off is the [K, num_output] table, num_output = out_shape.back()); the bottom holds
  // M = count(bottom) ids
  int64_t input_dim = 0;
  // RNN: x is [T, N, ...] (in_shape), the top [T, N, H]; bottoms[1] is cont [T, N] (the label-like bottom) and
  // bottoms[2], when there, x_static [N, ...].  The flat offsets of its blobs, by role: W_xh, b_h, W_xh_static (-1
  // without x_static), W_hh, W_ho, b_o.
  enum { kWxh, kBh, kWxhStatic, kWhh, kWho, kBo, kRnnBlobs };
  int64_t rnn_off[kRnnBlobs] = {-1, -1, -1, -1, -1, -1};
  // MVN: mvn_rows contiguous rows of mvn_dim elements each (num * channels rows, or num with across_channels), each
  // normalised on its own; eps is added to the standard deviation.  Mean-only without normalize_variance.
  int64_t mvn_rows = 0, mvn_dim = 0;
  bool normalize_variance = true, across_channels = false;
};

struct Plan {
  std::vector<Op> ops;
  std::vector<int64_t> tensor_count;   // elements per tensor id
  std::vector<int> storage;            // tensor id -> tensor id that owns its memory (itself unless in place)
  // per tensor id: its activation is another tensor's memory, set when the forward reaches it (a Split, Flatten or
  // Reshape top reads its bottom's, as Caffe's ShareData).  A Split top's gradient is still its own; a Flatten or
  // Reshape top's is its bottom's (storage, as Caffe's ShareDiff) unless the bottom is a staged input.
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
// ... of a MultinomialLogisticLoss or HingeLoss label outside [0, dim) (or NaN): its row adds no loss and gets a zero
// gradient
constexpr int kStatusBadMultinomialLabel = 501, kStatusBadHingeLabel = 502;
// ... of an Embed id that is not an integer in [0, input_dim) (negative, too large, fractional, NaN or infinite): its
// row embeds as the zero vector (plus the bias) and adds nothing to the weight gradient
constexpr int kStatusBadEmbedIndex = 503;
// PReLU's slope gradient runs one grid row per slope (gridDim.y), so a per-channel PReLU has at most this many channels
constexpr int64_t kMaxPReLUChannels = 65535;
// The GEMM core puts its M rows on gridDim.y in tiles of 64, so one GEMM has at most this many rows: an InnerProduct's
// rows or num_output, a convolution's input or output channels, an RNN's T * N or num_output
constexpr int64_t kMaxGemmRows = 65535 * 64;

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
                                          // BN save, MVN's per-row statistics (mvn.hpp)
  std::vector<float*> op_z_, op_dz_;      // fused block: conv output without bias and its gradient
  // per op, an RNN's buffers (null for other ops), all [rows, H] with rows as named: g = x W_xh^T + b_h (T N), z =
  // x_static W_xh_static^T (N), h = h_{-1} .. h_{T-1} ((T + 1) N), state = the hidden state carried from call to call
  // (N; zero at creation, h_{T-1} after every forward), dzo = the output tanh's input gradient (T N), dho = its
  // gradient at h (T N), dpre = the hidden tanh's input gradient (T N), dz = dpre summed over t (N)
  struct RnnBuffers {
    float *g = nullptr, *z = nullptr, *h = nullptr, *state = nullptr, *dzo = nullptr, *dho = nullptr,
          *dpre = nullptr, *dz = nullptr;
  };
  std::vector<RnnBuffers> rnn_;
  cudaEvent_t done_ = nullptr;            // recorded at the end of every call: the destructor waits for it
  float* workspace_ = nullptr;            // split-K partials, bias partials, BatchNorm scratch, the sigmoid
                                          // cross-entropy's per-block partials, Embed's id grouping (int32), MVN's
                                          // chunk partials (ops run in order)
  size_t workspace_floats_ = 0;
  std::vector<void*> allocations_;
};

}  // namespace cosb
#endif
