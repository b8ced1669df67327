// solver_spec.hpp -- what the hot path needs to know about the solver and the
// learnable-parameter layout.
//
// The reference obtains this from protobuf (SolverParameter, caffe.proto:102-;
// ParamSpec lr_mult/decay_mult :283-304) and from Net::learnable_params()
// after Caffe has built the net (parallel.cpp:27-57).  Here a small
// text-format reader plus shape inference over the layer types of the
// BASELINE configs recovers the same flat layout, so that
// CaffeNet.allocate(solver.prototxt, ...) keeps working unchanged.
#ifndef COS_SOLVER_SPEC_HPP_
#define COS_SOLVER_SPEC_HPP_

#include <cstdint>
#include <string>
#include <vector>

namespace cosb {

// FillerParameter (caffe.proto:43-62): what a weight_filler / bias_filler block says.  Caffe's default is constant 0.
struct FillerSpec {
  std::string type = "constant";
  float value = 0.f, min = 0.f, max = 1.f, mean = 0.f, std = 1.f;
  std::string variance_norm = "FAN_IN";
  int64_t sparse = -1;  // gaussian: keep each value with probability sparse / shape(0), as filler.hpp (-1: all)
};

// One TRAIN-phase layer as the layout parser saw it: its blobs' shapes (from the same shape inference that derives
// the learnable layout) and the parameters a forward/backward engine needs.  Fields a layer type does not have keep
// their defaults.
struct NetLayer {
  std::string name, type;
  std::vector<std::string> bottoms, tops;
  std::vector<std::vector<int64_t>> bottom_shapes, top_shapes;
  // per param of this layer: the learnable blob it reads (SolverSpec index; the owner's for a shared param), and
  // whether it is shared (a later use of a named param)
  std::vector<int> blobs;
  std::vector<bool> shared;
  // axis: InnerProduct's, Slice's, Concat's, Scale's, and SoftmaxWithLoss's class axis (softmax_param, canonical)
  int64_t num_output = 0, axis = 1, group = 1;
  int64_t kernel_h = 0, kernel_w = 0, stride_h = 1, stride_w = 1, pad_h = 0, pad_w = 0, dilation_h = 1, dilation_w = 1;
  // the depth axis of a Convolution or Deconvolution over a 5-axis bottom [N, C, D, H, W] (1, 1, 0, 1 otherwise).  One
  // over a 3-axis bottom [N, C, L] has kernel_h 1, stride_h 1 and pad_h 0: the 2-D layer over [N, C, 1, L].
  int64_t kernel_d = 1, stride_d = 1, pad_d = 0, dilation_d = 1;
  bool bias_term = true, transpose = false, global_pooling = false;
  std::string pool = "MAX";
  float negative_slope = 0.f;
  bool use_global_stats = false;  // BatchNorm in TRAIN: default false
  float moving_average_fraction = 0.999f, eps = 1e-5f;  // eps: BatchNorm's, or MVN's (the parser sets its 1e-9)
  // MVN (caffe.proto MVNParameter defaults)
  bool normalize_variance = true, across_channels = false;
  float loss_weight = 1.f;
  bool has_loss_param = false;
  // LRN (caffe.proto LRNParameter defaults); norm_region is "ACROSS_CHANNELS" or "WITHIN_CHANNEL"
  int64_t local_size = 5;
  float lrn_alpha = 1.f, lrn_beta = 0.75f, lrn_k = 1.f;
  std::string norm_region = "ACROSS_CHANNELS";
  // Slice (slice_layer.cpp): the canonical axis and every top's [begin, end) along it
  std::vector<int64_t> slice_begin, slice_end;
  // ContrastiveLoss (caffe.proto ContrastiveLossParameter)
  float margin = 1.f;
  bool legacy_version = false;
  // Scale (scale_layer.cpp): `axis` is the first scaled axis (0 when the scale is a scalar, as Reshape sets it) and
  // num_axes the scale's number of axes (-1 resolved); bias_term defaults to false here.  weight_filler is the scale's
  // filler (constant 1 when the prototxt gives none), bias_filler the bias's.
  int64_t num_axes = 1;
  // Eltwise (caffe.proto EltwiseParameter): "PROD", "SUM" or "MAX"; one coeff per bottom (all 1 when none are given)
  std::string eltwise_op = "SUM";
  std::vector<float> coeffs;
  bool stable_prod_grad = true;
  // Flatten (caffe.proto FlattenParameter) as written: flatten_axis and flatten_end_axis, negative counted from the end
  int64_t flatten_axis = 1, flatten_end_axis = -1;
  // Power, Exp and Log (caffe.proto PowerParameter, ExpParameter, LogParameter): power is Power's alone, base Exp's and
  // Log's (-1: e); scale and shift each layer's own
  float power = 1.f, scale = 1.f, shift = 0.f, base = -1.f;
  float elu_alpha = 1.f;   // ELUParameter
  float threshold = 0.f;   // ThresholdParameter
  // Softmax's softmax_param axis as written (negative counted from the end; the engine's plan checks it)
  int64_t softmax_axis = 1;
  bool channel_shared = false;  // PReLUParameter; its filler is weight_filler (constant 0.25 when none is given)
  std::string hinge_norm = "L1";  // HingeLossParameter: "L1" or "L2"
  // Embed (caffe.proto EmbedParameter): the vocabulary size; num_output, bias_term (default true) and the fillers are
  // the fields above
  int64_t input_dim = 0;
  // RNN (caffe.proto RecurrentParameter): num_output is H; bottoms x, cont and the optional x_static (a fourth bottom
  // and a second top with expose_hidden, which the parser lays out and the engine refuses)
  bool expose_hidden = false;
  bool static_input = false;
  // Crop (crop_layer.cpp): `axis` is the first cropped axis (canonical), and the offset of every axis of bottom[0]
  // (0 before `axis`)
  std::vector<int64_t> crop_offsets;
  // SPP (caffe.proto SPPParameter): the number of pyramid levels; `pool` is its pool method.  Level l's geometry is
  // spp_level()'s.
  int64_t pyramid_height = 0;
  // Tile (caffe.proto TileParameter): `axis` is the tiled axis (canonical), repeated `tiles` times
  int64_t tiles = 0;
  FillerSpec weight_filler, bias_filler;
  // per param: whether bias_filler fills it rather than weight_filler.  Empty for the layers whose params are a
  // weight and then (with bias_term) a bias.
  std::vector<bool> bias_param;
};

// A later use of a named param (net.cpp AppendParam): it reads the owner's data and adds its gradient into the owner's
// diff, and has no learnable blob, lr_mult or history of its own.
struct SharedParam {
  std::string layer_name, layer_type;
  int param_index = 0;  // index of the blob within its layer
  int owner = 0;        // the learnable blob it shares
  int position = 0;     // learnable blobs before it in net order: where Net::ToProto writes it among the owners
};

// TransformationParameter (caffe.proto) of one staged input: what Caffe's DataTransformer applies in TRAIN.  Only the
// path of a mean file is recorded here; data_transform.hpp reads it.
struct TransformSpec {
  bool present = false;  // the top has a transform_param
  float scale = 1.f;
  bool mirror = false;
  int64_t crop_size = 0;
  std::string mean_file;  // as written in the prototxt ("" = none)
  std::string net_file;   // the prototxt it was written in: a relative mean_file is also looked for next to it
  std::vector<float> mean_values;
};

// One staged input: a top of a data layer (MemoryData, CoSData, Input), in the order the producer receives them.
struct StagedInput {
  std::string layer, type, top;
  std::vector<int64_t> shape;
  TransformSpec transform;  // MemoryData: top 0 only; CoSData: each top's own
};

struct SolverSpec {
  // learnable blobs in learnable_params() order
  std::vector<int64_t> counts;
  std::vector<float> lr_mult, decay_mult;
  std::vector<std::string> blob_names;  // "<layer>.<index>" (diagnostics)
  // what Net::ToProto needs to write a stock-Caffe .caffemodel (solver.cpp:452-459)
  std::string net_name;
  std::vector<std::string> layer_names, layer_types;  // per learnable blob: owning layer
  std::vector<std::vector<int64_t>> shapes;            // per learnable blob: Blob shape
  std::vector<int> param_index;                        // per learnable blob: its index within its layer
  std::vector<SharedParam> shared;                     // every shared use of a named param, in net order
  bool snapshot_hdf5 = false;                          // SolverParameter.snapshot_format (caffe.proto:194-198)
  // SolverParameter
  std::string lr_policy = "fixed";
  float base_lr = 0.01f, gamma = 0.1f, power = 0.75f;
  int stepsize = 1;
  std::vector<int> stepvalues;
  int max_iter = 0;
  float momentum = 0.f, weight_decay = 0.f;
  int test_iter = 0, test_interval = 0;
  std::string snapshot_prefix;
  std::string regularization_type = "L2";
  std::string type = "SGD";
  int solver_type = 0;                   // COS_SOLVER_SGD / COS_SOLVER_ADAM (from type)
  float momentum2 = 0.999f, delta = 1e-8f;  // Adam's beta2 and epsilon (caffe.proto:213-218); momentum is beta1
  int iter_size = 1;
  float clip_gradients = -1.f;
  bool solver_mode_gpu = true;
  int64_t random_seed = -1;  // SolverParameter.random_seed (caffe.proto: default -1)
  std::string solver_file;   // the solver prototxt this spec was parsed from ("" for a descriptor)
  // training input layer
  int batch_size = 0;
  std::vector<int> input_shape;  // N,C,H,W of the first top of the data layer
  std::vector<StagedInput> inputs;  // every staged input with its transform_param (empty for a descriptor)
  // this library's extensions
  int grad_dtype = 0;  // COS_GRAD_FP32 / COS_GRAD_BF16
  int init_iter = 0;

  uint64_t param_count() const;  // max(1, sum counts): parallel.cpp:60-68
  // history blobs per learnable blob: 1 for SGD, 2 for Adam (AdamPreSolve appends v, adam_solver.cpp:8-17)
  int history_sets() const { return solver_type == 1 ? 2 : 1; }
};

// Blob::count(from): the product of the axes from `from` on (1 for none).
int64_t shape_count(const std::vector<int64_t>& s, size_t from = 0);
// "2x3x4", or "scalar" for a shape without axes.
std::string shape_text(const std::vector<int64_t>& s);

// SPPLayer::GetPoolingParam: level l of a pyramid over a height x width map pools bins = 2^l windows per side, with
// kernel k = ceil(height / bins), stride k and pad (k bins - height + 1) / 2 (the same for the width).
struct SppLevel {
  int64_t bins, kernel_h, kernel_w, pad_h, pad_w;
};
SppLevel spp_level(int64_t height, int64_t width, int level);

// SocketSync::chunk (socket_sync_cpu.cpp:46-54).
void chunk(uint64_t param_count, int cluster_size, int peer, uint64_t* offs, uint64_t* size);

// Adam's bias correction sqrt(1 - beta2^t) / (1 - beta1^t) for t = iter + 1 (adam_solver.cpp:39-41): pow with a
// float base and an int exponent is the double pow, so the whole expression is double, rounded once to float.
float adam_correction(float beta1, float beta2, int iter);

// SGDSolver::GetLearningRate (sgd_solver.cpp:27-63), Dtype = float.
// Returns false for an unknown policy.
bool learning_rate(const std::string& policy, float base_lr, float gamma, float power, int stepsize,
                   const int* stepvalues, int nstepvalues, int max_iter, int iter, int* current_step,
                   float* rate);

// Parses a solver prototxt and the net it references (net:, train_net: or
// inline net_param/train_net_param) and fills `spec`.
bool parse_solver_prototxt(const std::string& solver_path, SolverSpec* spec, std::string* err);
// Checks that apply once the layout is known: an Adam solver needs at least one learnable element (a snapshot of a
// net without any holds no history blobs, so restore could not refuse a state of the other solver kind).
bool check_solver_layout(const SolverSpec& spec, std::string* err);
// A solver prototxt (its net is read as parse_solver_prototxt reads it) or a net prototxt, told apart by whether the
// file has top-level layers: fills spec (solver fields only for a solver file) and the TRAIN-phase layer list.
bool parse_train_net(const std::string& path, SolverSpec* spec, std::vector<NetLayer>* layers, std::string* err);
// The file `path` names, looked for as the solver's net: path is: as given, then relative to the directory of
// `relative_to`, then by its basename in that directory.  "" when none can be opened.
std::string find_relative_file(const std::string& path, const std::string& relative_to);

}  // namespace cosb
#endif
