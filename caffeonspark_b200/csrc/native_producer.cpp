// native_producer.cpp -- the built-in producer's net plan (host only); see native_producer.hpp.
#include "native_producer.hpp"

#include <cmath>
#include <map>
#include <sstream>

#include "caffe_layers.hpp"

namespace cosb {
namespace {

bool is_data_layer(const std::string& t) { return t == "MemoryData" || t == "CoSData" || t == "Input"; }

std::string why(const NetLayer& L, const std::string& reason) {
  return "layer '" + L.name + "' (" + L.type + "): " + reason + " (native producer)";
}

int64_t count_of(const std::vector<int64_t>& s) {
  int64_t n = 1;
  for (int64_t d : s) n *= d;
  return n;
}

std::string shape_str(const std::vector<int64_t>& s) {
  std::ostringstream os;
  for (size_t i = 0; i < s.size(); ++i) os << (i ? "x" : "") << s[i];
  return s.empty() ? "scalar" : os.str();
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
  return true;
}

// Caffe's ReLU and MAX pool as the existing fused block accepts them: slope 0; square window, pad 0, kernel <= 15.
bool fusable_relu(const NetLayer& L) {
  return L.type == "ReLU" && L.negative_slope == 0.f && L.bottoms.size() == 1 && L.tops.size() == 1;
}
bool fusable_pool(const NetLayer& L) {
  return L.type == "Pooling" && L.pool == "MAX" && !L.global_pooling && L.pad_h == 0 && L.pad_w == 0 &&
         L.kernel_h == L.kernel_w && L.stride_h == L.stride_w && L.kernel_h <= 15 && L.bottoms.size() == 1 &&
         L.tops.size() == 1 && L.bottom_shapes[0].size() == 4;
}

// The weight (and bias) of a Convolution or InnerProduct: a shared param uses its owner's offsets, and only the owner's
// filler fills the blob.
void set_params(const NetLayer& L, Op* op, Plan* P) {
  op->w_off = P->blob_off[L.blobs[0]], op->w_count = P->blob_count[L.blobs[0]];
  if (!L.shared[0]) P->blob_filler[L.blobs[0]] = L.weight_filler;
  if (L.bias_term) {
    op->b_off = P->blob_off[L.blobs[1]], op->b_count = P->blob_count[L.blobs[1]];
    if (!L.shared[1]) P->blob_filler[L.blobs[1]] = L.bias_filler;
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
      cur[L.tops[t]] = new_tensor(count_of(L.top_shapes[t]), -1);
      P.input_names.push_back(L.tops[t]);
    }
  }
  P.ninputs = static_cast<int>(P.tensor_count.size());
  int losses = 0;
  for (size_t i = 0; i < layers.size(); ++i) {
    const NetLayer& L = layers[i];
    if (is_data_layer(L.type) || L.type == "Accuracy" || L.type == "Silence") continue;  // no TRAIN work
    if (L.has_loss_param) {
      *err = why(L, "loss_param is not supported (only the default VALID normalisation without ignore_label is)");
      return false;
    }
    const bool known = L.type == "Convolution" || L.type == "Pooling" || L.type == "InnerProduct" || L.type == "ReLU" ||
                       L.type == "Sigmoid" || L.type == "BatchNorm" || L.type == "SoftmaxWithLoss" ||
                       L.type == "Slice" || L.type == "ContrastiveLoss" || L.type == "Concat" ||
                       L.type == "EuclideanLoss" || L.type == "Split" || L.type == "Eltwise" || L.type == "Scale" ||
                       (L.type == "LRN" && L.norm_region == "WITHIN_CHANNEL");  // ACROSS_CHANNELS has no engine op
    if (!known) {
      *err = why(L, "layer type not supported");
      return false;
    }
    if (L.type == "Scale" && L.bottoms.size() == 2) {
      *err = why(L, "the two-bottom form (the scale read from bottom[1]) is not supported");
      return false;
    }
    // Slice and Split are the layers with several tops, Concat and Eltwise the ones with any number of bottoms (the
    // parser checked Eltwise's at least 2); ContrastiveLoss reads a, b and sim.  EuclideanLoss may leave its top out,
    // as Caffe's solver tests write it (a loss layer's AutoTopBlobs): the engine writes the loss to loss_dev either way.
    const size_t want_bottoms = L.type == "SoftmaxWithLoss" || L.type == "EuclideanLoss" ? 2
                                : L.type == "ContrastiveLoss"                             ? 3
                                                                                          : 1;
    const bool any_bottoms = L.type == "Concat" || L.type == "Eltwise";
    const bool auto_top = L.type == "EuclideanLoss" && L.tops.empty();
    const bool tops_ok = L.type == "Slice" || L.type == "Split" ? !L.tops.empty() : L.tops.size() == 1 || auto_top;
    if ((any_bottoms ? L.bottoms.empty() : L.bottoms.size() != want_bottoms) || !tops_ok) {
      *err = why(L, (any_bottoms ? std::string("needs at least 1") : std::to_string(want_bottoms)) +
                        " bottom(s) and one top");
      return false;
    }
    Op op;
    op.name = L.name;
    for (size_t j = 0; j < L.blobs.size(); ++j)
      if (L.shared[j]) op.shares.push_back(L.blobs[j]);
    auto take = [&](const std::string& name, int* id) {
      auto it = cur.find(name);
      if (it == cur.end()) {
        *err = why(L, "bottom '" + name + "' is not produced by an earlier TRAIN layer");
        return false;
      }
      if (!consumer[it->second].empty()) {
        *err = why(L, "bottom '" + name + "' already feeds layer '" + consumer[it->second] +
                          "'; a blob read by two layers needs a Split");
        return false;
      }
      consumer[it->second] = L.name;
      *id = it->second;
      return true;
    };
    if (!take(L.bottoms[0], &op.in)) return false;
    op.in_shape = L.bottom_shapes[0];
    if (!auto_top) op.out_shape = L.top_shapes[0];  // else the scalar loss
    op.need_dx = wants_grad[op.in];
    if (L.type == "Slice") {  // one op per top, each copying its range of the bottom (and back, in the backward)
      op.kind = OpKind::kSlice;
      op.slice_axis = static_cast<int>(L.axis);
      for (size_t t = 0; t < L.tops.size(); ++t) {
        op.slice_begin = L.slice_begin[t];
        op.out_shape = L.top_shapes[t];
        op.out = new_tensor(count_of(op.out_shape), -1);
        wants_grad[op.out] = op.need_dx;
        cur[L.tops[t]] = op.out;
        P.ops.push_back(op);
      }
      continue;
    }
    if (L.type == "Split") {  // one op per top; each top reads the bottom's activation (split_layer.cpp ShareData)
      op.kind = OpKind::kSplit;
      for (size_t t = 0; t < L.tops.size(); ++t) {
        op.split_top = static_cast<int>(t);
        op.out = new_tensor(count_of(op.out_shape), -1);
        P.data_alias[op.out] = true;
        wants_grad[op.out] = op.need_dx;
        cur[L.tops[t]] = op.out;
        P.ops.push_back(op);
      }
      continue;
    }
    if (L.type == "Eltwise") {  // eltwise_layer.cpp: every bottom is consumed, the top has storage of its own
      op.kind = OpKind::kEltwise;
      op.eltwise_op = L.eltwise_op == "PROD" ? kEltwiseProd : L.eltwise_op == "MAX" ? kEltwiseMax : kEltwiseSum;
      op.coeffs = L.coeffs;
      op.stable_prod_grad = L.stable_prod_grad;
      op.ins = {op.in};
      op.ins_need_dx = {op.need_dx};
      for (size_t b = 1; b < L.bottoms.size(); ++b) {
        int id;
        if (!take(L.bottoms[b], &id)) return false;
        op.ins.push_back(id);
        op.ins_need_dx.push_back(wants_grad[id]);
      }
      op.out = new_tensor(count_of(op.out_shape), -1);
      for (bool need : op.ins_need_dx) wants_grad[op.out] = wants_grad[op.out] || need;
      cur[L.tops[0]] = op.out;
      P.ops.push_back(op);
      continue;
    }
    if (L.type == "Concat") {  // one op per bottom, each copying its bottom into its range of the one top (and back)
      op.kind = OpKind::kConcat;
      op.slice_axis = static_cast<int>(L.axis);  // the parser checked the axis and the bottoms' shapes
      op.out = new_tensor(count_of(op.out_shape), -1);
      int64_t begin = 0;
      for (size_t b = 0; b < L.bottoms.size(); ++b) {
        if (b > 0) {
          if (!take(L.bottoms[b], &op.in)) return false;
          op.in_shape = L.bottom_shapes[b];
          op.need_dx = wants_grad[op.in];
        }
        op.slice_begin = begin;
        begin += op.in_shape[op.slice_axis];
        wants_grad[op.out] = wants_grad[op.out] || op.need_dx;
        P.ops.push_back(op);
      }
      cur[L.tops[0]] = op.out;
      continue;
    }
    int storage = -1;
    std::string reason;
    if (L.type == "Convolution") {
      if (L.group != 1) {
        *err = why(L, "group " + std::to_string(L.group) + " > 1 is not supported");
        return false;
      }
      if (L.dilation_h != 1 || L.dilation_w != 1) {
        *err = why(L, "dilation other than 1 is not supported");
        return false;
      }
      if (!filler_ok(L.weight_filler, &reason) || (L.bias_term && !filler_ok(L.bias_filler, &reason))) {
        *err = why(L, reason);
        return false;
      }
      op.kind = OpKind::kConv;
      op.kh = static_cast<int>(L.kernel_h), op.kw = static_cast<int>(L.kernel_w);
      op.sh = static_cast<int>(L.stride_h), op.sw = static_cast<int>(L.stride_w);
      op.ph = static_cast<int>(L.pad_h), op.pw = static_cast<int>(L.pad_w);
      set_params(L, &op, &P);
      // conv + bias followed by ReLU and MAX pool in either order: the existing fused block (caffe_layers.cu)
      if (L.bias_term && i + 2 < layers.size()) {
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
            const int out = new_tensor(count_of(op.out_shape), -1);
            wants_grad[out] = true;  // the block has a weight and a bias
            cur[b.tops[0]] = out;
            op.out = out;
            P.ops.push_back(op);
            i += 2;
            continue;
          }
        }
      }
    } else if (L.type == "Pooling") {
      if (L.pool != "MAX" && L.pool != "AVE") {
        *err = why(L, "pool method " + L.pool + " is not supported (MAX and AVE are)");
        return false;
      }
      op.kind = OpKind::kPool;
      op.max_pool = L.pool == "MAX";
      op.kh = static_cast<int>(L.kernel_h), op.kw = static_cast<int>(L.kernel_w);
      op.sh = static_cast<int>(L.stride_h), op.sw = static_cast<int>(L.stride_w);
      op.ph = static_cast<int>(L.pad_h), op.pw = static_cast<int>(L.pad_w);
    } else if (L.type == "InnerProduct") {
      if (L.transpose) {
        *err = why(L, "transpose: true is not supported");
        return false;
      }
      if (L.axis != 1) {
        *err = why(L, "axis other than 1 is not supported");
        return false;
      }
      if (!filler_ok(L.weight_filler, &reason) || (L.bias_term && !filler_ok(L.bias_filler, &reason))) {
        *err = why(L, reason);
        return false;
      }
      op.kind = OpKind::kInnerProduct;
      set_params(L, &op, &P);
    } else if (L.type == "ReLU" || L.type == "Sigmoid") {
      op.kind = L.type == "ReLU" ? OpKind::kReLU : OpKind::kSigmoid;
      op.slope = L.negative_slope;
      // top == bottom shares the bottom's memory, except on a staged input: that is never written (every pass of an
      // iter_size step reads it again), so the top gets storage of its own.  So does a Split top: its memory is the
      // Split's bottom, which the sibling tops read too.
      op.in_place = L.tops[0] == L.bottoms[0] && op.in >= P.ninputs && !P.data_alias[op.in];
      if (op.in_place) storage = P.storage[op.in];
    } else if (L.type == "BatchNorm") {
      if (!op.shares.empty()) {
        *err = why(L, "shared BatchNorm statistics are not supported");
        return false;
      }
      op.kind = OpKind::kBatchNorm;  // separate top storage even when top == bottom: the kernels are not in place
      op.w_off = P.blob_off[L.blobs[0]];
      op.global_stats = L.use_global_stats;
      op.fraction = L.moving_average_fraction;
      op.eps = L.eps;
    } else if (L.type == "Scale") {  // scale_layer.cpp, one-bottom form; the parser resolved axis and num_axes
      if (!filler_ok(L.weight_filler, &reason) || (L.bias_term && !filler_ok(L.bias_filler, &reason))) {
        *err = why(L, reason);
        return false;
      }
      op.kind = OpKind::kScale;  // separate top storage even when top == bottom: the scale's gradient reads x
      set_params(L, &op, &P);
      const size_t first = static_cast<size_t>(L.axis), end = first + static_cast<size_t>(L.num_axes);
      op.scale_outer = count_of(std::vector<int64_t>(op.in_shape.begin(), op.in_shape.begin() + first));
      op.scale_dim = count_of(std::vector<int64_t>(op.in_shape.begin() + first, op.in_shape.begin() + end));
      op.scale_inner = count_of(std::vector<int64_t>(op.in_shape.begin() + end, op.in_shape.end()));
    } else if (L.type == "LRN") {
      if (L.local_size < 1 || L.local_size % 2 == 0 || L.local_size > kLrnMaxLocalSize) {
        *err = why(L, "local_size " + std::to_string(L.local_size) + " is not odd and <= " +
                          std::to_string(kLrnMaxLocalSize));
        return false;
      }
      if (op.in_shape.size() != 4 || !std::isfinite(L.lrn_beta)) {
        *err = why(L, "needs a 4-axis bottom and a finite beta");
        return false;
      }
      op.kind = OpKind::kLRNWithin;  // separate top storage even when top == bottom: the kernels read a halo
      op.lrn_size = static_cast<int>(L.local_size);
      op.lrn_alpha = L.lrn_alpha;
      op.lrn_beta = L.lrn_beta;
    } else if (L.type == "ContrastiveLoss") {  // the parser checked the shapes: a, b N x C (x 1 x 1), sim N values
      if (++losses > 1) {
        *err = why(L, "a second loss layer is not supported");
        return false;
      }
      op.kind = OpKind::kContrastiveLoss;
      op.loss_weight = L.loss_weight;
      op.margin = L.margin;
      op.legacy = L.legacy_version;
      if (!take(L.bottoms[1], &op.in2)) return false;
      op.need_dx2 = wants_grad[op.in2];
      auto it = cur.find(L.bottoms[2]);
      if (it == cur.end()) {
        *err = why(L, "sim bottom '" + L.bottoms[2] + "' is not produced by an earlier TRAIN layer");
        return false;
      }
      op.label = it->second;
    } else if (L.type == "EuclideanLoss") {  // euclidean_loss_layer.cpp, after LossLayer::Reshape's check
      if (++losses > 1) {
        *err = why(L, "a second loss layer is not supported");
        return false;
      }
      const std::vector<int64_t>& a = L.bottom_shapes[0];
      const std::vector<int64_t>& b = L.bottom_shapes[1];
      if (a.empty() || b.empty() || a[0] != b[0]) {
        *err = why(L, "The data and label should have the same number.");
        return false;
      }
      if (count_of(std::vector<int64_t>(a.begin() + 1, a.end())) !=
          count_of(std::vector<int64_t>(b.begin() + 1, b.end()))) {  // Blob::count(1)
        *err = why(L, "Inputs must have the same dimension.");
        return false;
      }
      op.kind = OpKind::kEuclideanLoss;
      op.loss_weight = L.loss_weight;
      if (!take(L.bottoms[1], &op.in2)) return false;
      op.need_dx2 = wants_grad[op.in2];
    } else {  // SoftmaxWithLoss
      if (++losses > 1) {
        *err = why(L, "a second loss layer is not supported");
        return false;
      }
      op.kind = OpKind::kSoftmaxLoss;
      op.loss_weight = L.loss_weight;
      auto it = cur.find(L.bottoms[1]);
      if (it == cur.end()) {
        *err = why(L, "label bottom '" + L.bottoms[1] + "' is not produced by an earlier TRAIN layer");
        return false;
      }
      op.label = it->second;
      const int64_t rows = op.in_shape.empty() ? 0 : count_of(op.in_shape) / (op.in_shape.size() > 1 ? op.in_shape[1] : 1);
      if (op.in_shape.size() < 2 || P.tensor_count[op.label] != rows) {
        *err = why(L, "label count " + std::to_string(P.tensor_count[op.label]) + " does not match the " +
                          std::to_string(rows) + " rows of the scores");
        return false;
      }
    }
    op.out = new_tensor(count_of(op.out_shape), storage);
    // BatchNorm's blobs are statistics, with no gradient
    wants_grad[op.out] = op.need_dx || (op.kind != OpKind::kBatchNorm && (op.w_off >= 0 || op.b_off >= 0));
    if (!auto_top) cur[L.tops[0]] = op.out;
    P.ops.push_back(op);
  }
  // the op of each Split's top 0 sums the gradients of the tops some layer reads (consumer[] is complete now)
  for (size_t i = 0; i < P.ops.size(); ++i) {
    if (P.ops[i].kind != OpKind::kSplit || P.ops[i].split_top != 0) continue;
    for (size_t j = i; j < P.ops.size() && P.ops[j].kind == OpKind::kSplit && P.ops[j].in == P.ops[i].in; ++j) {
      if (j > i && P.ops[j].split_top == 0) break;  // the next Split of the same bottom
      if (consumer[P.ops[j].out].empty()) P.ops[j].split_unread = true;
      else P.ops[i].split_sum.push_back(P.ops[j].out);
    }
  }
  if (losses == 0) {
    *err = "the net has no SoftmaxWithLoss, ContrastiveLoss or EuclideanLoss layer in its TRAIN phase (native producer)";
    return false;
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
  static const char* kinds[] = {"Convolution", "ConvBiasReLUMaxPool", "Pooling", "InnerProduct",
                                "ReLU",        "Sigmoid",             "BatchNorm", "SoftmaxWithLoss",
                                "LRN(WITHIN_CHANNEL)", "Slice", "ContrastiveLoss", "Concat", "EuclideanLoss",
                                "Split", "Eltwise", "Scale"};
  static const char* eltwise_ops[] = {"PROD", "SUM", "MAX"};
  std::ostringstream os;
  for (int i = 0; i < ninputs; ++i) os << "input " << i << " " << input_names[i] << " " << tensor_count[i] << "\n";
  for (size_t i = 0; i < ops.size(); ++i) {
    const Op& op = ops[i];
    os << "op " << i << " " << kinds[static_cast<int>(op.kind)];
    if (op.kind == OpKind::kPool) os << "(" << (op.max_pool ? "MAX" : "AVE") << ")";
    if (op.kind == OpKind::kEltwise) os << "(" << eltwise_ops[op.eltwise_op] << ")";
    os << " " << op.name << " " << shape_str(op.in_shape) << " -> " << shape_str(op.out_shape);
    if (op.kind == OpKind::kConv || op.kind == OpKind::kConvBiasReluMaxPool || op.kind == OpKind::kPool)
      os << " k" << op.kh << "x" << op.kw << " s" << op.sh << "x" << op.sw << " p" << op.ph << "x" << op.pw;
    if (op.kind == OpKind::kConvBiasReluMaxPool) os << " pool" << op.pool_kernel << "/" << op.pool_stride;
    if (op.kind == OpKind::kReLU && op.slope != 0.f) os << " slope=" << op.slope;
    if (op.kind == OpKind::kLRNWithin) os << " n=" << op.lrn_size << " alpha=" << op.lrn_alpha << " beta=" << op.lrn_beta;
    if (op.w_off >= 0 && op.kind != OpKind::kBatchNorm) os << " w=" << op.w_off << ":" << op.w_count;
    if (op.b_off >= 0) os << " b=" << op.b_off << ":" << op.b_count;
    if (op.kind == OpKind::kBatchNorm) os << " stats=" << op.w_off;
    if (!op.shares.empty()) {
      os << " shares=";
      for (size_t j = 0; j < op.shares.size(); ++j) os << (j ? "," : "") << op.shares[j];
    }
    if (op.kind == OpKind::kSlice || op.kind == OpKind::kConcat)
      os << " axis=" << op.slice_axis << " begin=" << op.slice_begin;
    if (op.kind == OpKind::kSoftmaxLoss) os << " label=" << op.label << " loss_weight=" << op.loss_weight;
    if (op.kind == OpKind::kContrastiveLoss)
      os << " second=" << op.in2 << " sim=" << op.label << " margin=" << op.margin << (op.legacy ? " legacy" : "")
         << " loss_weight=" << op.loss_weight;
    if (op.kind == OpKind::kEuclideanLoss) os << " second=" << op.in2 << " loss_weight=" << op.loss_weight;
    if (op.kind == OpKind::kSplit) os << " top=" << op.split_top << " data=bottom" << (op.split_unread ? " unread" : "");
    if (op.kind == OpKind::kEltwise) {
      os << " bottoms=" << op.ins.size();
      if (op.eltwise_op == kEltwiseSum) {
        os << " coeff=";
        for (size_t j = 0; j < op.coeffs.size(); ++j) os << (j ? "," : "") << op.coeffs[j];
      }
      if (op.eltwise_op == kEltwiseProd) os << (op.stable_prod_grad ? " stable_prod_grad" : " top/bottom_grad");
    }
    if (op.kind == OpKind::kScale)
      os << " outer=" << op.scale_outer << " dim=" << op.scale_dim << " inner=" << op.scale_inner;
    if (op.in_place) os << " in-place";
    // no data gradient is propagated into a staged input, nor into a blob with no learnable blob before it
    auto mark = [&](int in, bool need) { return need ? "" : in < ninputs ? " staged-bottom" : " no-bottom-grad"; };
    const char* m = mark(op.in, op.need_dx);
    if (!*m && (op.kind == OpKind::kContrastiveLoss || op.kind == OpKind::kEuclideanLoss)) m = mark(op.in2, op.need_dx2);
    for (size_t j = 1; j < op.ins.size() && !*m; ++j) m = mark(op.ins[j], op.ins_need_dx[j]);  // Eltwise
    os << m;
    os << "\n";
  }
  os << "params " << param_count << " blobs " << blob_count.size() << "\n";
  for (size_t k = 0; k < blob_off.size(); ++k)
    os << "blob " << k << " " << blob_off[k] << ":" << blob_count[k] << " " << shape_str(blob_shape[k]) << " "
       << blob_filler[k].type << "\n";
  return os.str();
}

}  // namespace cosb
