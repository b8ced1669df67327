// native_producer.cpp -- the built-in producer's net plan (host only); see native_producer.hpp.
#include "native_producer.hpp"

#include <algorithm>
#include <cmath>
#include <iterator>
#include <map>
#include <sstream>

#include "caffe_layers.hpp"

namespace cosb {
namespace {

bool is_data_layer(const std::string& t) { return t == "MemoryData" || t == "CoSData" || t == "Input"; }

std::string why(const NetLayer& L, const std::string& reason) {
  return "layer '" + L.name + "' (" + L.type + "): " + reason + " (native producer)";
}

bool filler_ok(const FillerSpec& f, std::string* reason) {
  static const char* types[] = {"constant", "uniform", "gaussian", "xavier", "msra"};
  bool known = false;
  for (const char* t : types) known = known || f.type == t;
  if (!known) {
    *reason = "filler type '" + f.type + "' is not supported (constant, uniform, gaussian, xavier, msra are)";
    return false;
  }
  if (f.variance_norm != "FAN_IN" && f.variance_norm != "FAN_OUT" && f.variance_norm != "AVERAGE") {
    *reason = "filler variance_norm '" + f.variance_norm + "' is not FAN_IN, FAN_OUT or AVERAGE";
    return false;
  }
  if (f.sparse != -1 && (f.type != "gaussian" || f.sparse < -1)) {  // filler.hpp's CHECKs
    *reason = f.type != "gaussian" ? "Sparsity not supported by this Filler." : "Check failed: sparse >= -1";
    return false;
  }
  return true;
}

// Caffe's ReLU and MAX pool as the existing fused block accepts them: slope 0; square window, pad 0, kernel <= 15, and
// no empty window.  Caffe's pooled size ceil((H - k) / s) + 1 (pad 0: no clip) counts a last window that starts at or
// past the edge when s >= k + r (H - k = q * s + r, 0 < r < s); ReLU then MAX pool writes -FLT_MAX there, while the
// fused block pools only the pooled_size() windows, which all start inside.  So it fuses only when the two sizes agree.
bool fusable_relu(const NetLayer& L) {
  return L.type == "ReLU" && L.negative_slope == 0.f && L.bottoms.size() == 1 && L.tops.size() == 1;
}
bool fusable_pool(const NetLayer& L) {
  if (L.type != "Pooling" || L.pool != "MAX" || L.global_pooling || L.pad_h != 0 || L.pad_w != 0 ||
      L.kernel_h != L.kernel_w || L.stride_h != L.stride_w || L.kernel_h > 15 || L.bottoms.size() != 1 ||
      L.tops.size() != 1 || L.bottom_shapes[0].size() != 4 || L.top_shapes[0].size() != 4)
    return false;
  const int k = static_cast<int>(L.kernel_h), s = static_cast<int>(L.stride_h);
  return L.top_shapes[0][2] == pooled_size(static_cast<int>(L.bottom_shapes[0][2]), k, s) &&
         L.top_shapes[0][3] == pooled_size(static_cast<int>(L.bottom_shapes[0][3]), k, s);
}

// The weight (and bias) of a Convolution, Deconvolution, InnerProduct, Scale or Embed: a shared param uses its owner's
// offsets, and only the owner's filler fills the blob.  False when a filler is one the engine cannot draw.
bool set_params(const NetLayer& L, Op* op, Plan* P, std::string* err) {
  std::string reason;
  if (!filler_ok(L.weight_filler, &reason) || (L.bias_term && !filler_ok(L.bias_filler, &reason))) {
    *err = why(L, reason);
    return false;
  }
  op->w_off = P->blob_off[L.blobs[0]], op->w_count = P->blob_count[L.blobs[0]];
  if (!L.shared[0]) P->blob_filler[L.blobs[0]] = L.weight_filler;
  if (L.bias_term) {
    op->b_off = P->blob_off[L.blobs[1]], op->b_count = P->blob_count[L.blobs[1]];
    if (!L.shared[1]) P->blob_filler[L.blobs[1]] = L.bias_filler;
  }
  return true;
}

// LossLayer::Reshape's check, then euclidean_loss_layer.cpp's or sigmoid_cross_entropy_loss_layer.cpp's: the two
// bottoms hold as many values (per item, or in all: the same once the numbers agree), with the layer's own wording
bool loss_shapes_ok(const NetLayer& L, const char* count_message, std::string* err) {
  const std::vector<int64_t>& a = L.bottom_shapes[0];
  const std::vector<int64_t>& b = L.bottom_shapes[1];
  if (a.empty() || b.empty() || a[0] != b[0]) {
    *err = why(L, "The data and label should have the same number.");
    return false;
  }
  if (shape_count(a, 1) != shape_count(b, 1)) {
    *err = why(L, count_message);
    return false;
  }
  return true;
}

// The layer types the engine runs.  bottoms: the exact count, or -1 for any number from 1 (the parser checked
// Eltwise's at least 2).  several_tops: one op per top.  label: the label-like bottom (read, never differentiated and
// not counted as its blob's reader), called `role` in refusals, or -1.  loss: a net has one loss layer.
struct LayerType {
  const char* type;
  OpKind kind;
  int bottoms = 1;
  bool several_tops = false;
  int label = -1;
  const char* role = nullptr;
  bool loss = false;
};
const LayerType kLayerTypes[] = {
    {"Convolution", OpKind::kConv},
    {"Pooling", OpKind::kPool},
    {"InnerProduct", OpKind::kInnerProduct},
    {"ReLU", OpKind::kReLU},
    {"Sigmoid", OpKind::kSigmoid},
    {"BatchNorm", OpKind::kBatchNorm},
    {"LRN", OpKind::kLRNWithin},  // WITHIN_CHANNEL only: ACROSS_CHANNELS has no engine op
    {"Slice", OpKind::kSlice, 1, true},
    {"Split", OpKind::kSplit, 1, true},
    {"Concat", OpKind::kConcat, -1},
    {"Eltwise", OpKind::kEltwise, -1},
    {"Scale", OpKind::kScale},  // the one-bottom form
    {"Deconvolution", OpKind::kDeconv},
    {"Flatten", OpKind::kFlatten},  // axis 1 to the end only
    {"SoftmaxWithLoss", OpKind::kSoftmaxLoss, 2, false, 1, "label", true},
    {"ContrastiveLoss", OpKind::kContrastiveLoss, 3, false, 2, "sim", true},  // a, b, sim
    {"EuclideanLoss", OpKind::kEuclideanLoss, 2, false, -1, nullptr, true},
    {"SigmoidCrossEntropyLoss", OpKind::kSigmoidCrossEntropyLoss, 2, false, 1, "target", true},
    // the other neuron layers, Softmax and the classification losses; none shares memory with its bottom
    {"TanH", OpKind::kTanH},
    {"ELU", OpKind::kELU},
    {"AbsVal", OpKind::kAbsVal},
    {"BNLL", OpKind::kBNLL},
    {"Power", OpKind::kPower},
    {"Exp", OpKind::kExp},
    {"Log", OpKind::kLog},
    {"Threshold", OpKind::kThreshold},  // forward only: refused where a gradient would have to pass it
    {"PReLU", OpKind::kPReLU},
    {"Softmax", OpKind::kSoftmax},
    {"MultinomialLogisticLoss", OpKind::kMultinomialLogisticLoss, 2, false, 1, "label", true},
    {"HingeLoss", OpKind::kHingeLoss, 2, false, 1, "label", true},
    {"Embed", OpKind::kEmbed},      // its bottom's ids get no gradient
    {"Reshape", OpKind::kReshape},  // Flatten's alias: no copy either way
    // x, cont and the optional x_static (the parser checked the count); cont is read, never differentiated, so two
    // RNNs may read one cont blob
    {"RNN", OpKind::kRNN, -1, false, 1, "cont"},
    {"MVN", OpKind::kMVN},
};

// Plan::text's name of each OpKind
const char* const kKindNames[] = {"Convolution", "ConvBiasReLUMaxPool", "Pooling", "InnerProduct", "ReLU", "Sigmoid",
                                  "BatchNorm", "SoftmaxWithLoss", "LRN(WITHIN_CHANNEL)", "Slice", "ContrastiveLoss",
                                  "Concat", "EuclideanLoss", "Split", "Eltwise", "Scale", "Deconvolution", "Flatten",
                                  "SigmoidCrossEntropyLoss", "TanH", "ELU", "AbsVal", "BNLL", "Power", "Exp", "Log",
                                  "Threshold", "PReLU", "Softmax", "MultinomialLogisticLoss", "HingeLoss",
                                  "Embed", "Reshape", "RNN", "MVN"};
static_assert(std::size(kKindNames) == static_cast<size_t>(OpKind::kCount), "one name per OpKind");

// LossLayer::Reshape's check, then multinomial_logistic_loss_layer.cpp's: the label holds one value per item, with
// Blob::channels(), height() and width() all 1 (mll only)
bool label_shapes_ok(const NetLayer& L, bool mll, std::string* err) {
  const std::vector<int64_t>& a = L.bottom_shapes[0];
  const std::vector<int64_t>& b = L.bottom_shapes[1];
  if (a.empty() || b.empty() || a[0] != b[0]) {
    *err = why(L, "The data and label should have the same number.");
    return false;
  }
  static const char* legacy[] = {"channels", "height", "width"};
  for (size_t k = 1; mll && k < 4; ++k) {
    const int64_t v = k < b.size() ? b[k] : 1;  // Blob::LegacyShape
    if (v != 1) {
      *err = why(L, std::string("Check failed: bottom[1]->") + legacy[k - 1] + "() == 1 (" + std::to_string(v) +
                        " vs. 1)");
      return false;
    }
  }
  return true;
}

std::string float_text(float v) {
  std::ostringstream os;
  os << v;
  return os.str();
}

// The neuron ops, Softmax and the two classification losses: their parameters as Caffe's LayerSetUp derives them (in
// float), and its refusals.  None shares memory with its bottom, in place or not.  True for every other kind.
bool neuron_op(const NetLayer& L, Op* op, Plan* P, std::string* err) {
  switch (op->kind) {
    case OpKind::kELU:
      op->alpha = L.elu_alpha;
      return true;
    case OpKind::kAbsVal:
      if (L.tops[0] == L.bottoms[0]) {
        *err = why(L, "AbsVal Layer does not allow in-place computation.");
        return false;
      }
      return true;
    case OpKind::kPower:
      op->power = L.power, op->scale = L.scale, op->shift = L.shift;
      return true;
    case OpKind::kExp:
    case OpKind::kLog: {  // exp_layer.cpp, log_layer.cpp
      op->base = L.base, op->scale = L.scale, op->shift = L.shift;
      if (L.base != -1.f && !(L.base > 0.f)) {
        *err = why(L, "base must be strictly positive.");
        return false;
      }
      const float log_base = L.base == -1.f ? 1.f : std::log(L.base);
      if (!std::isfinite(log_base)) {
        *err = why(L, "Inf result: log(base) = log(" + float_text(L.base) + ") = " + float_text(log_base));
        return false;
      }
      if (op->kind == OpKind::kExp) {
        op->inner_scale = log_base * L.scale;
        op->outer_scale = L.shift == 0.f ? 1.f : L.base != -1.f ? std::pow(L.base, L.shift) : std::exp(L.shift);
        return true;
      }
      op->base_scale = 1.f / log_base;
      if (!std::isfinite(op->base_scale)) {
        *err = why(L, "Inf result: 1/log(base) = 1/log(" + float_text(L.base) + ") = " + float_text(op->base_scale));
        return false;
      }
      op->backward_num_scale = L.scale / log_base;
      return true;
    }
    case OpKind::kThreshold:
      op->threshold = L.threshold;
      return true;
    case OpKind::kPReLU: {  // prelu_layer.cpp: one slope per channel of axis 1, or one for the whole blob
      if (op->in_shape.size() < 2) {
        *err = why(L, "Number of axes of bottom blob must be >=2.");
        return false;
      }
      std::string reason;
      if (!filler_ok(L.weight_filler, &reason)) {
        *err = why(L, reason);
        return false;
      }
      op->w_off = P->blob_off[L.blobs[0]], op->w_count = P->blob_count[L.blobs[0]];
      if (!L.shared[0]) P->blob_filler[L.blobs[0]] = L.weight_filler;
      op->channel_shared = L.channel_shared;
      op->prelu_channels = op->in_shape[1];
      if (!L.channel_shared && op->prelu_channels > kMaxPReLUChannels) {  // the slope gradient's gridDim.y
        *err = why(L, std::to_string(op->prelu_channels) + " channels is more than the " +
                          std::to_string(kMaxPReLUChannels) + " per-channel slopes the engine supports");
        return false;
      }
      op->prelu_dim = shape_count(op->in_shape, 2);
      return true;
    }
    case OpKind::kSoftmax: {  // softmax_layer.cpp Reshape: CanonicalAxisIndex(softmax_param.axis)
      const int64_t naxes = static_cast<int64_t>(op->in_shape.size());
      const int64_t axis = L.softmax_axis < 0 ? L.softmax_axis + naxes : L.softmax_axis;
      if (axis < 0 || axis >= naxes) {
        *err = why(L, "axis " + std::to_string(L.softmax_axis) + " out of range for " + std::to_string(naxes) +
                          "-D Blob");
        return false;
      }
      op->softmax_axis = static_cast<int>(axis);
      op->classes = op->in_shape[axis];
      op->inner = shape_count(op->in_shape, axis + 1);
      op->outer = shape_count(std::vector<int64_t>(op->in_shape.begin(), op->in_shape.begin() + axis));
      return true;
    }
    case OpKind::kHingeLoss:
      if (L.hinge_norm != "L1" && L.hinge_norm != "L2") {
        *err = why(L, "Unknown Norm");
        return false;
      }
      op->hinge_l2 = L.hinge_norm == "L2";
      return true;
    default:
      return true;
  }
}

// The largest M of the op's GEMMs (0 for an op without one): the channels of a convolution's forward and data gradient
// (either side, as a Deconvolution swaps them), an InnerProduct's rows (forward, data gradient) and num_output (weight
// gradient), an RNN's T * N rows and its num_output
int64_t gemm_rows(const Op& op) {
  switch (op.kind) {
    case OpKind::kConv:
    case OpKind::kConvBiasReluMaxPool:
    case OpKind::kDeconv:
      return std::max(op.in_shape[1], op.out_shape[1]);
    case OpKind::kInnerProduct:
      return std::max(shape_count(op.out_shape) / op.out_shape.back(), op.out_shape.back());
    case OpKind::kRNN:
      return std::max(op.in_shape[0] * op.in_shape[1], op.out_shape[2]);
    default:
      return 0;
  }
}

}  // namespace

bool build_plan(const SolverSpec& spec, const std::vector<NetLayer>& layers, Plan* plan, std::string* err) {
  Plan P;
  int64_t off = 0;
  for (size_t k = 0; k < spec.counts.size(); ++k) {
    P.blob_off.push_back(off);
    P.blob_count.push_back(spec.counts[k]);
    P.blob_shape.push_back(k < spec.shapes.size() ? spec.shapes[k] : std::vector<int64_t>{spec.counts[k]});
    P.blob_filler.push_back(FillerSpec());
    off += spec.counts[k];
  }
  P.param_count = off;
  std::map<std::string, int> cur;  // blob name -> tensor id it currently names
  std::vector<std::string> consumer;  // per tensor: the layer that reads it ("" = none yet)
  // per tensor: whether anything before it has a learnable blob, so that its gradient is wanted (Caffe's
  // bottom_need_backward).  Staged inputs want none.
  std::vector<bool> wants_grad;
  auto new_tensor = [&](int64_t n, int storage) {
    P.tensor_count.push_back(n);
    P.storage.push_back(storage < 0 ? static_cast<int>(P.tensor_count.size()) - 1 : storage);
    P.data_alias.push_back(false);
    consumer.emplace_back();
    wants_grad.push_back(false);
    return static_cast<int>(P.tensor_count.size()) - 1;
  };
  for (const NetLayer& L : layers) {  // staged inputs first: tensors 0 .. ninputs-1
    if (!is_data_layer(L.type)) continue;
    for (size_t t = 0; t < L.tops.size(); ++t) {
      cur[L.tops[t]] = new_tensor(shape_count(L.top_shapes[t]), -1);
      P.input_names.push_back(L.tops[t]);
    }
  }
  P.ninputs = static_cast<int>(P.tensor_count.size());
  int losses = 0;
  int loss_top = -1;  // the loss layer's top: never written, the loss goes to loss_dev
  std::string loss_layer;
  for (size_t i = 0; i < layers.size(); ++i) {
    const NetLayer& L = layers[i];
    if (is_data_layer(L.type) || L.type == "Accuracy" || L.type == "Silence") continue;  // no TRAIN work
    const LayerType* row = nullptr;
    for (const LayerType& r : kLayerTypes)
      if (L.type == r.type) row = &r;
    // Net::Init gives a loss layer of weight 0 no backward, and its value never reaches the objective: no TRAIN work
    // either (a monitor such as the MNIST autoencoder's l2_error), so its bottoms do not count as read
    if (row && row->loss && L.loss_weight == 0.f) continue;
    if (L.has_loss_param) {
      *err = why(L, "loss_param is not supported (only the default VALID normalisation without ignore_label is)");
      return false;
    }
    if (!row || (row->kind == OpKind::kLRNWithin && L.norm_region != "WITHIN_CHANNEL")) {
      *err = why(L, "layer type not supported");
      return false;
    }
    if (row->kind == OpKind::kRNN && L.expose_hidden) {
      *err = why(L, "expose_hidden: true is not supported");
      return false;
    }
    if (row->kind == OpKind::kScale && L.bottoms.size() == 2) {
      *err = why(L, "the two-bottom form (the scale read from bottom[1]) is not supported");
      return false;
    }
    // EuclideanLoss may leave its top out, as Caffe's solver tests write it (a loss layer's AutoTopBlobs): the engine
    // writes the loss to loss_dev either way.
    const bool auto_top = row->kind == OpKind::kEuclideanLoss && L.tops.empty();
    const bool tops_ok = row->several_tops ? !L.tops.empty() : L.tops.size() == 1 || auto_top;
    if ((row->bottoms < 0 ? L.bottoms.empty() : L.bottoms.size() != static_cast<size_t>(row->bottoms)) || !tops_ok) {
      *err = why(L, (row->bottoms < 0 ? std::string("needs at least 1") : std::to_string(row->bottoms)) +
                        " bottom(s) and one top");
      return false;
    }
    Op op;
    op.kind = row->kind;
    op.name = L.name;
    op.label_bottom = row->label;
    op.in_shape = L.bottom_shapes[0];
    if (!auto_top) op.out_shape = L.top_shapes[0];  // else the scalar loss
    if (row->loss) op.loss_weight = L.loss_weight;
    for (size_t j = 0; j < L.blobs.size(); ++j)
      if (L.shared[j]) op.shares.push_back(L.blobs[j]);
    bool top_grad = false;  // the top wants a gradient when a bottom does (or, below, when the op has a weight or bias)
    for (size_t b = 0; b < L.bottoms.size(); ++b) {
      const std::string& name = L.bottoms[b];
      const bool label = static_cast<int>(b) == row->label;
      auto it = cur.find(name);
      if (it == cur.end()) {
        *err = why(L, (label ? std::string(row->role) + " " : std::string()) + "bottom '" + name +
                          "' is not produced by an earlier TRAIN layer");
        return false;
      }
      const int id = it->second;
      if (id == loss_top) {
        *err = why(L, "bottom '" + name + "' is the top of loss layer '" + loss_layer +
                          "'; reading a loss layer's top is not supported");
        return false;
      }
      if (!label) {
        if (!consumer[id].empty()) {
          *err = why(L, "bottom '" + name + "' already feeds layer '" + consumer[id] +
                            "'; a blob read by two layers needs a Split");
          return false;
        }
        consumer[id] = L.name;
      }
      op.bottoms.push_back(id);
      op.bottom_grad.push_back(!label && wants_grad[id]);
      top_grad = top_grad || op.bottom_grad.back();
      if (b > 0 || !row->loss) continue;
      // a loss layer's own checks come after its first bottom, before the others
      if (++losses > 1) {
        *err = why(L, "a second loss layer is not supported");
        return false;
      }
      if (row->kind == OpKind::kEuclideanLoss && !loss_shapes_ok(L, "Inputs must have the same dimension.", err))
        return false;
      if (row->kind == OpKind::kSigmoidCrossEntropyLoss &&
          !loss_shapes_ok(L, "SIGMOID_CROSS_ENTROPY_LOSS layer inputs must have the same count.", err))
        return false;
      if ((row->kind == OpKind::kMultinomialLogisticLoss || row->kind == OpKind::kHingeLoss) &&
          !label_shapes_ok(L, row->kind == OpKind::kMultinomialLogisticLoss, err))
        return false;
    }
    if (op.kind == OpKind::kSlice) {  // one op per top, each copying its range of the bottom (and back, in the backward)
      op.slice_axis = static_cast<int>(L.axis);
      for (size_t t = 0; t < L.tops.size(); ++t) {
        op.slice_begin = L.slice_begin[t];
        op.out_shape = L.top_shapes[t];
        op.out = new_tensor(shape_count(op.out_shape), -1);
        wants_grad[op.out] = top_grad;
        cur[L.tops[t]] = op.out;
        P.ops.push_back(op);
      }
      continue;
    }
    if (op.kind == OpKind::kSplit) {  // one op per top; each top reads the bottom's activation (split_layer.cpp ShareData)
      for (size_t t = 0; t < L.tops.size(); ++t) {
        op.split_top = static_cast<int>(t);
        op.out = new_tensor(shape_count(op.out_shape), -1);
        P.data_alias[op.out] = true;
        wants_grad[op.out] = top_grad;
        cur[L.tops[t]] = op.out;
        P.ops.push_back(op);
      }
      continue;
    }
    if (op.kind == OpKind::kConcat) {  // one op per bottom, each copying its bottom into its range of the one top (and back)
      op.slice_axis = static_cast<int>(L.axis);  // the parser checked the axis and the bottoms' shapes
      op.out = new_tensor(shape_count(op.out_shape), -1);
      wants_grad[op.out] = top_grad;
      int64_t begin = 0;
      for (size_t b = 0; b < L.bottoms.size(); ++b) {
        Op part = op;
        part.bottoms = {op.bottoms[b]};
        part.bottom_grad = {op.bottom_grad[b]};
        part.in_shape = L.bottom_shapes[b];
        part.slice_begin = begin;
        begin += part.in_shape[op.slice_axis];
        P.ops.push_back(part);
      }
      cur[L.tops[0]] = op.out;
      continue;
    }
    int storage = -1;
    const std::string* top = auto_top ? nullptr : &L.tops[0];
    if (op.kind == OpKind::kConv || op.kind == OpKind::kDeconv) {
      if (L.group != 1) {
        *err = why(L, "group " + std::to_string(L.group) + " > 1 is not supported");
        return false;
      }
      if (L.dilation_h != 1 || L.dilation_w != 1) {
        *err = why(L, "dilation other than 1 is not supported");
        return false;
      }
      if (!set_params(L, &op, &P, err)) return false;
      op.kh = static_cast<int>(L.kernel_h), op.kw = static_cast<int>(L.kernel_w);
      op.sh = static_cast<int>(L.stride_h), op.sw = static_cast<int>(L.stride_w);
      op.ph = static_cast<int>(L.pad_h), op.pw = static_cast<int>(L.pad_w);
      // conv + bias followed by ReLU and MAX pool in either order: the existing fused block (caffe_layers.cu)
      if (op.kind == OpKind::kConv && L.bias_term && i + 2 < layers.size()) {
        const NetLayer& a = layers[i + 1];
        const NetLayer& b = layers[i + 2];
        const bool order = (fusable_relu(a) && fusable_pool(b)) || (fusable_pool(a) && fusable_relu(b));
        if (order && a.bottoms[0] == L.tops[0] && b.bottoms[0] == a.tops[0]) {
          bool private_mid = true;  // the intermediates must not be read by any later layer
          for (size_t j = i + 3; j < layers.size(); ++j)
            for (const std::string& bn : layers[j].bottoms)
              if ((bn == L.tops[0] || bn == a.tops[0]) && bn != b.tops[0]) private_mid = false;
          if (private_mid) {
            const NetLayer& pool = a.type == "Pooling" ? a : b;
            op.kind = OpKind::kConvBiasReluMaxPool;
            op.name = L.name + "+" + a.name + "+" + b.name;
            op.pool_kernel = static_cast<int>(pool.kernel_h);
            op.pool_stride = static_cast<int>(pool.stride_h);
            op.out_shape = b.top_shapes[0];
            top = &b.tops[0];
            i += 2;
          }
        }
      }
    } else if (op.kind == OpKind::kPool) {
      if (L.pool != "MAX" && L.pool != "AVE") {
        *err = why(L, "pool method " + L.pool + " is not supported (MAX and AVE are)");
        return false;
      }
      op.max_pool = L.pool == "MAX";
      op.kh = static_cast<int>(L.kernel_h), op.kw = static_cast<int>(L.kernel_w);
      op.sh = static_cast<int>(L.stride_h), op.sw = static_cast<int>(L.stride_w);
      op.ph = static_cast<int>(L.pad_h), op.pw = static_cast<int>(L.pad_w);
    } else if (op.kind == OpKind::kInnerProduct) {
      if (L.transpose) {
        *err = why(L, "transpose: true is not supported");
        return false;
      }
      // inner_product_layer.cpp: count(0, axis) rows of K = count(axis) inputs each; the parser made the axis canonical
      const int64_t naxes = static_cast<int64_t>(op.in_shape.size());
      if (L.axis >= naxes) {
        *err = why(L, "axis " + std::to_string(L.axis) + " out of range for " + std::to_string(naxes) + "-D Blob");
        return false;
      }
      if (!set_params(L, &op, &P, err)) return false;
    } else if (op.kind == OpKind::kReLU || op.kind == OpKind::kSigmoid) {
      op.slope = L.negative_slope;
      // top == bottom shares the bottom's memory, except on a staged input: that is never written (every pass of an
      // iter_size step reads it again), so the top gets storage of its own.  So does a Split top: its memory is the
      // Split's bottom, which the sibling tops read too.
      const int in = op.bottoms[0];
      op.in_place = L.tops[0] == L.bottoms[0] && in >= P.ninputs && !P.data_alias[in];
      if (op.in_place) storage = P.storage[in];
    } else if (op.kind == OpKind::kFlatten || op.kind == OpKind::kReshape) {
      // flatten_layer.cpp, reshape_layer.cpp: no copy either way (ShareData, ShareDiff); the parser inferred the shape
      if (L.tops[0] == L.bottoms[0]) {
        *err = why(L, L.type + " Layer does not allow in-place computation.");
        return false;
      }
      const int64_t naxes = static_cast<int64_t>(op.in_shape.size());
      const int64_t first = L.flatten_axis < 0 ? L.flatten_axis + naxes : L.flatten_axis;
      const int64_t last = L.flatten_end_axis < 0 ? L.flatten_end_axis + naxes : L.flatten_end_axis;
      if (op.kind == OpKind::kFlatten && (first != 1 || last != naxes - 1)) {
        *err = why(L, "flatten_param axis " + std::to_string(L.flatten_axis) + ", end_axis " +
                          std::to_string(L.flatten_end_axis) + " is not supported (axis 1 to the last axis is)");
        return false;
      }
      // the top's gradient is the bottom's, except on a staged input, whose gradient buffer nothing may share
      const int in = op.bottoms[0];
      if (in >= P.ninputs) storage = P.storage[in];
    } else if (op.kind == OpKind::kEmbed) {  // embed_layer.cpp: a gather of table rows; ids have no derivative
      if (op.bottom_grad[0]) {
        *err = why(L, "Can't backpropagate to EmbedLayer input.");
        return false;
      }
      if (!set_params(L, &op, &P, err)) return false;
      op.input_dim = L.input_dim;
    } else if (op.kind == OpKind::kRNN) {  // recurrent_layer.cpp, rnn_layer.cpp; the parser checked the shapes
      std::string reason;
      if (!filler_ok(L.weight_filler, &reason) || !filler_ok(L.bias_filler, &reason)) {
        *err = why(L, reason);
        return false;
      }
      // the layer's params in the parser's order; W_xh_static only with x_static
      std::vector<int> roles = {Op::kWxh, Op::kBh, Op::kWhh, Op::kWho, Op::kBo};
      if (L.static_input) roles.insert(roles.begin() + 2, Op::kWxhStatic);
      for (size_t j = 0; j < roles.size(); ++j) {
        op.rnn_off[roles[j]] = P.blob_off[L.blobs[j]];
        if (!L.shared[j]) P.blob_filler[L.blobs[j]] = L.bias_param[j] ? L.bias_filler : L.weight_filler;
      }
    } else if (op.kind == OpKind::kMVN) {  // mvn_layer.cpp; the parser gave the top the bottom's legacy 4-D shape
      // The top gets storage of its own even when top == bottom, unlike Caffe: its in-place Backward_gpu overwrites
      // top_diff with y * dy and then sums that again as if it were dy (DESIGN.md section 14)
      op.normalize_variance = L.normalize_variance;
      op.across_channels = L.across_channels;
      op.eps = L.eps;
      op.mvn_rows = op.out_shape[0] * (L.across_channels ? 1 : op.out_shape[1]);
      op.mvn_dim = shape_count(op.out_shape) / op.mvn_rows;
    } else if (op.kind == OpKind::kBatchNorm) {
      if (!op.shares.empty()) {
        *err = why(L, "shared BatchNorm statistics are not supported");
        return false;
      }
      // separate top storage even when top == bottom: the kernels are not in place
      op.w_off = P.blob_off[L.blobs[0]];
      op.global_stats = L.use_global_stats;
      op.fraction = L.moving_average_fraction;
      op.eps = L.eps;
    } else if (op.kind == OpKind::kEltwise) {  // eltwise_layer.cpp: the top has storage of its own
      op.eltwise_op = L.eltwise_op == "PROD" ? kEltwiseProd : L.eltwise_op == "MAX" ? kEltwiseMax : kEltwiseSum;
      op.coeffs = L.coeffs;
      op.stable_prod_grad = L.stable_prod_grad;
    } else if (op.kind == OpKind::kScale) {  // scale_layer.cpp, one-bottom form; the parser resolved axis and num_axes
      // separate top storage even when top == bottom: the scale's gradient reads x
      if (!set_params(L, &op, &P, err)) return false;
      const size_t first = static_cast<size_t>(L.axis), end = first + static_cast<size_t>(L.num_axes);
      op.scale_outer = shape_count(std::vector<int64_t>(op.in_shape.begin(), op.in_shape.begin() + first));
      op.scale_dim = shape_count(std::vector<int64_t>(op.in_shape.begin() + first, op.in_shape.begin() + end));
      op.scale_inner = shape_count(op.in_shape, end);
    } else if (op.kind == OpKind::kLRNWithin) {
      if (L.local_size < 1 || L.local_size % 2 == 0 || L.local_size > kLrnMaxLocalSize) {
        *err = why(L, "local_size " + std::to_string(L.local_size) + " is not odd and <= " +
                          std::to_string(kLrnMaxLocalSize));
        return false;
      }
      if (op.in_shape.size() != 4 || !std::isfinite(L.lrn_beta)) {
        *err = why(L, "needs a 4-axis bottom and a finite beta");
        return false;
      }
      // separate top storage even when top == bottom: the kernels read a halo
      op.lrn_size = static_cast<int>(L.local_size);
      op.lrn_alpha = L.lrn_alpha;
      op.lrn_beta = L.lrn_beta;
    } else if (!neuron_op(L, &op, &P, err)) {
      return false;
    } else if (op.kind == OpKind::kContrastiveLoss) {  // the parser checked the shapes: a, b N x C (x 1 x 1), sim N values
      op.margin = L.margin;
      op.legacy = L.legacy_version;
    } else if (op.kind == OpKind::kSoftmaxLoss) {  // the parser made the axis canonical for the scores' shape
      const size_t axis = static_cast<size_t>(L.axis);
      if (L.axis < 0 || axis >= op.in_shape.size()) {
        *err = why(L, "axis " + std::to_string(L.axis) + " is not an axis of the " + shape_text(op.in_shape) + " scores");
        return false;
      }
      op.softmax_axis = static_cast<int>(axis);
      op.classes = op.in_shape[axis];
      op.inner = shape_count(op.in_shape, axis + 1);
      op.rows = shape_count(std::vector<int64_t>(op.in_shape.begin(), op.in_shape.begin() + axis)) * op.inner;
      const int64_t labels = P.tensor_count[op.bottoms[1]];
      if (labels != op.rows) {
        *err = why(L, "label count " + std::to_string(labels) + " does not match the " + std::to_string(op.rows) +
                          " rows of the scores along axis " + std::to_string(axis));
        return false;
      }
    }
    const int64_t rows = gemm_rows(op);
    if (rows > kMaxGemmRows) {
      *err = why(L, "a GEMM of " + std::to_string(rows) + " rows is more than the " + std::to_string(kMaxGemmRows) +
                        " the engine supports");
      return false;
    }
    op.out = new_tensor(shape_count(op.out_shape), storage);
    if (op.kind == OpKind::kFlatten || op.kind == OpKind::kReshape) P.data_alias[op.out] = true;
    // BatchNorm's blobs are statistics, with no gradient
    wants_grad[op.out] = top_grad || op.kind == OpKind::kRNN ||
                         (op.kind != OpKind::kBatchNorm && (op.w_off >= 0 || op.b_off >= 0));
    if (top) cur[*top] = op.out;
    if (row->loss) loss_top = op.out, loss_layer = L.name;
    P.ops.push_back(op);
  }
  if (losses == 0) {
    *err = "the net has no SoftmaxWithLoss, ContrastiveLoss, EuclideanLoss or SigmoidCrossEntropyLoss layer with a "
           "non-zero loss_weight in its TRAIN phase (native producer)";
    return false;
  }
  // Caffe's blobs_under_loss: the loss's top, and every non-label bottom of an op whose top is under the loss.  Every
  // blob has one reader (Splits aside), so one pass in reverse order finds them.  An op whose top is not under the loss
  // runs no backward; a Split top that is not adds nothing to its bottom's gradient, and a Slice top's op still writes
  // its range of the bottom's gradient (zeros), which the other ranges' readers need.
  std::vector<bool> under_loss(P.tensor_count.size(), false);
  under_loss[loss_top] = true;
  for (size_t i = P.ops.size(); i-- > 0;) {
    Op& op = P.ops[i];
    if (!under_loss[op.out]) {
      if (op.kind == OpKind::kSplit) op.split_unread = true;
      else if (op.kind != OpKind::kSlice) op.no_backward = true;
      continue;
    }
    for (size_t b = 0; b < op.bottoms.size(); ++b)
      if (static_cast<int>(b) != op.label_bottom) under_loss[op.bottoms[b]] = true;
  }
  // threshold_layer.cpp has no backward: a Threshold runs only where Caffe never calls it (its top off the loss, or no
  // gradient wanted at its bottom), such as one that binarises a staged target
  for (const Op& op : P.ops) {
    if (op.kind == OpKind::kThreshold && !op.no_backward && op.bottom_grad[0]) {
      *err = "layer '" + op.name + "' (Threshold): Not Implemented Yet: Threshold has no backward, and a gradient "
             "reaches it and is wanted at its bottom (native producer)";
      return false;
    }
  }
  // recurrent_layer.cpp Backward_cpu: an RNN under the loss whose cont would get a gradient (Caffe's propagate_down[1])
  for (const Op& op : P.ops) {
    if (op.kind == OpKind::kRNN && !op.no_backward && wants_grad[op.bottoms[1]]) {
      *err = "layer '" + op.name + "' (RNN): Cannot backpropagate to sequence indicators. (native producer)";
      return false;
    }
  }
  // the op of each Split's top 0 sums the gradients of the tops under the loss, in top order
  for (size_t i = 0; i < P.ops.size(); ++i) {
    if (P.ops[i].kind != OpKind::kSplit || P.ops[i].split_top != 0) continue;
    for (size_t j = i; j < P.ops.size() && P.ops[j].kind == OpKind::kSplit && P.ops[j].bottoms[0] == P.ops[i].bottoms[0];
         ++j) {
      if (j > i && P.ops[j].split_top == 0) break;  // the next Split of the same bottom
      if (!P.ops[j].split_unread) P.ops[i].split_sum.push_back(P.ops[j].out);
    }
  }
  for (size_t t = 0; t < P.tensor_count.size(); ++t) {
    if (P.tensor_count[t] <= 0 || P.tensor_count[t] >= (int64_t(1) << 31)) {
      *err = "a blob of " + std::to_string(P.tensor_count[t]) + " elements is outside the native producer's range";
      return false;
    }
  }
  *plan = std::move(P);
  return true;
}

bool plan_from_prototxt(const std::string& path, SolverSpec* spec, Plan* plan, std::string* err) {
  std::vector<NetLayer> layers;
  return parse_train_net(path, spec, &layers, err) && build_plan(*spec, layers, plan, err);
}

std::string Plan::text() const {
  static const char* eltwise_ops[] = {"PROD", "SUM", "MAX"};
  std::ostringstream os;
  for (int i = 0; i < ninputs; ++i) os << "input " << i << " " << input_names[i] << " " << tensor_count[i] << "\n";
  for (size_t i = 0; i < ops.size(); ++i) {
    const Op& op = ops[i];
    os << "op " << i << " " << kKindNames[static_cast<int>(op.kind)];
    if (op.kind == OpKind::kPool) os << "(" << (op.max_pool ? "MAX" : "AVE") << ")";
    if (op.kind == OpKind::kEltwise) os << "(" << eltwise_ops[op.eltwise_op] << ")";
    os << " " << op.name << " " << shape_text(op.in_shape) << " -> " << shape_text(op.out_shape);
    if (op.kind == OpKind::kConv || op.kind == OpKind::kConvBiasReluMaxPool || op.kind == OpKind::kPool ||
        op.kind == OpKind::kDeconv)
      os << " k" << op.kh << "x" << op.kw << " s" << op.sh << "x" << op.sw << " p" << op.ph << "x" << op.pw;
    if (op.kind == OpKind::kConvBiasReluMaxPool) os << " pool" << op.pool_kernel << "/" << op.pool_stride;
    if (op.kind == OpKind::kReLU && op.slope != 0.f) os << " slope=" << op.slope;
    if (op.kind == OpKind::kLRNWithin) os << " n=" << op.lrn_size << " alpha=" << op.lrn_alpha << " beta=" << op.lrn_beta;
    if (op.kind == OpKind::kEmbed) os << " input_dim=" << op.input_dim << " num_output=" << op.out_shape.back();
    if (op.kind == OpKind::kRNN) {
      static const char* roles[] = {"w_xh", "b_h", "w_xh_static", "w_hh", "w_ho", "b_o"};
      os << " T=" << op.in_shape[0] << " N=" << op.in_shape[1] << " H=" << op.out_shape[2] << " cont=" << op.bottoms[1];
      if (op.bottoms.size() > 2) os << " static=" << op.bottoms[2];
      for (int r = 0; r < Op::kRnnBlobs; ++r)
        if (op.rnn_off[r] >= 0) os << " " << roles[r] << "=" << op.rnn_off[r];
    }
    if (op.kind == OpKind::kMVN) {
      os << " rows=" << op.mvn_rows << " dim=" << op.mvn_dim << " eps=" << op.eps;
      if (op.across_channels) os << " across";
      if (!op.normalize_variance) os << " mean-only";
    }
    if (op.w_off >= 0 && op.kind != OpKind::kBatchNorm) os << " w=" << op.w_off << ":" << op.w_count;
    if (op.b_off >= 0) os << " b=" << op.b_off << ":" << op.b_count;
    if (op.kind == OpKind::kBatchNorm) os << " stats=" << op.w_off;
    if (!op.shares.empty()) {
      os << " shares=";
      for (size_t j = 0; j < op.shares.size(); ++j) os << (j ? "," : "") << op.shares[j];
    }
    if (op.kind == OpKind::kSlice || op.kind == OpKind::kConcat)
      os << " axis=" << op.slice_axis << " begin=" << op.slice_begin;
    if (op.kind == OpKind::kSoftmaxLoss)
      os << " axis=" << op.softmax_axis << " label=" << op.bottoms[1] << " loss_weight=" << op.loss_weight;
    if (op.kind == OpKind::kContrastiveLoss)
      os << " second=" << op.bottoms[1] << " sim=" << op.bottoms[2] << " margin=" << op.margin
         << (op.legacy ? " legacy" : "") << " loss_weight=" << op.loss_weight;
    if (op.kind == OpKind::kEuclideanLoss) os << " second=" << op.bottoms[1] << " loss_weight=" << op.loss_weight;
    if (op.kind == OpKind::kSigmoidCrossEntropyLoss)
      os << " target=" << op.bottoms[1] << " loss_weight=" << op.loss_weight;
    if (op.kind == OpKind::kFlatten || op.kind == OpKind::kReshape)
      os << " data=bottom" << (storage[op.out] != op.out ? " diff=bottom" : "");
    if (op.kind == OpKind::kSplit) os << " top=" << op.split_top << " data=bottom" << (op.split_unread ? " unread" : "");
    if (op.kind == OpKind::kEltwise) {
      os << " bottoms=" << op.bottoms.size();
      if (op.eltwise_op == kEltwiseSum) {
        os << " coeff=";
        for (size_t j = 0; j < op.coeffs.size(); ++j) os << (j ? "," : "") << op.coeffs[j];
      }
      if (op.eltwise_op == kEltwiseProd) os << (op.stable_prod_grad ? " stable_prod_grad" : " top/bottom_grad");
    }
    if (op.kind == OpKind::kScale)
      os << " outer=" << op.scale_outer << " dim=" << op.scale_dim << " inner=" << op.scale_inner;
    if (op.kind == OpKind::kELU) os << " alpha=" << op.alpha;
    if (op.kind == OpKind::kPower) os << " power=" << op.power << " scale=" << op.scale << " shift=" << op.shift;
    if (op.kind == OpKind::kExp || op.kind == OpKind::kLog)
      os << " base=" << op.base << " scale=" << op.scale << " shift=" << op.shift;
    if (op.kind == OpKind::kThreshold) os << " threshold=" << op.threshold;
    if (op.kind == OpKind::kPReLU && op.channel_shared) os << " channel_shared";
    if (op.kind == OpKind::kSoftmax) os << " axis=" << op.softmax_axis;
    if (op.kind == OpKind::kMultinomialLogisticLoss) os << " label=" << op.bottoms[1] << " loss_weight=" << op.loss_weight;
    if (op.kind == OpKind::kHingeLoss)
      os << " label=" << op.bottoms[1] << " norm=" << (op.hinge_l2 ? "L2" : "L1") << " loss_weight=" << op.loss_weight;
    if (op.in_place) os << " in-place";
    // the first bottom that gets no data gradient: a staged input, or a blob with no learnable blob before it
    for (size_t j = 0; j < op.bottoms.size(); ++j) {
      if (op.bottom_grad[j] || static_cast<int>(j) == op.label_bottom) continue;
      os << (op.bottoms[j] < ninputs ? " staged-bottom" : " no-bottom-grad");
      break;
    }
    if (op.no_backward) os << " no-backward";
    os << "\n";
  }
  os << "params " << param_count << " blobs " << blob_count.size() << "\n";
  for (size_t k = 0; k < blob_off.size(); ++k)
    os << "blob " << k << " " << blob_off[k] << ":" << blob_count[k] << " " << shape_text(blob_shape[k]) << " "
       << blob_filler[k].type << "\n";
  return os.str();
}

}  // namespace cosb
