// solver_spec.cpp -- see solver_spec.hpp.
#include "solver_spec.hpp"

#include <math.h>
#include <stdlib.h>

#include <fstream>
#include <map>
#include <memory>
#include <sstream>

namespace cosb {

uint64_t SolverSpec::param_count() const {
  uint64_t n = 0;
  for (int64_t c : counts) n += static_cast<uint64_t>(c);
  return n > 0 ? n : 1;  // "Size have at least one byte" (parallel.cpp:66-67)
}

// socket_sync_cpu.cpp:46-54: size_t arithmetic, multiply before divide.
void chunk(uint64_t param_count, int cluster_size, int peer, uint64_t* offs, uint64_t* size) {
  const uint64_t n = static_cast<uint64_t>(cluster_size);
  const uint64_t start = (static_cast<uint64_t>(peer) + 0) * param_count / n;
  const uint64_t until = (static_cast<uint64_t>(peer) + 1) * param_count / n;
  *offs = start;
  *size = until - start;
}

// sgd_solver.cpp:27-63 with Dtype = float.  The reference's unqualified
// pow()/exp() take float sub-expressions, evaluate in double and the product
// with base_lr is rounded to float when assigned to `Dtype rate`.
float adam_correction(float beta1, float beta2, int iter) {
  const int t = iter + 1;
  return static_cast<float>(sqrt(1.0 - pow(static_cast<double>(beta2), t)) /
                            (1.0 - pow(static_cast<double>(beta1), t)));
}

bool learning_rate(const std::string& policy, float base_lr, float gamma, float power, int stepsize,
                   const int* stepvalues, int nstepvalues, int max_iter, int iter, int* current_step,
                   float* rate) {
  if (policy == "fixed") {
    *rate = base_lr;
  } else if (policy == "step") {
    if (stepsize <= 0) return false;
    *current_step = iter / stepsize;
    *rate = static_cast<float>(static_cast<double>(base_lr) *
                               pow(static_cast<double>(gamma), static_cast<double>(*current_step)));
  } else if (policy == "exp") {
    *rate = static_cast<float>(static_cast<double>(base_lr) *
                               pow(static_cast<double>(gamma), static_cast<double>(iter)));
  } else if (policy == "inv") {
    const float base = 1.0f + gamma * static_cast<float>(iter);
    const float e = -power;
    *rate = static_cast<float>(static_cast<double>(base_lr) * pow(static_cast<double>(base), static_cast<double>(e)));
  } else if (policy == "multistep") {
    if (*current_step < nstepvalues && iter >= stepvalues[*current_step]) (*current_step)++;
    *rate = static_cast<float>(static_cast<double>(base_lr) *
                               pow(static_cast<double>(gamma), static_cast<double>(*current_step)));
  } else if (policy == "poly") {
    const float base = 1.0f - (static_cast<float>(iter) / static_cast<float>(max_iter));
    *rate = static_cast<float>(static_cast<double>(base_lr) *
                               pow(static_cast<double>(base), static_cast<double>(power)));
  } else if (policy == "sigmoid") {
    const float x = -gamma * (static_cast<float>(iter) - static_cast<float>(stepsize));
    const double d = 1.0 / (1.0 + exp(static_cast<double>(x)));
    *rate = static_cast<float>(static_cast<double>(base_lr) * d);
  } else {
    return false;  // LOG(FATAL) << "Unknown learning rate policy" (:60)
  }
  return true;
}

int64_t shape_count(const std::vector<int64_t>& s, size_t from) {
  int64_t n = 1;
  for (size_t i = from; i < s.size(); ++i) n *= s[i];
  return n;
}

std::string shape_text(const std::vector<int64_t>& s) {
  std::string t;
  for (size_t i = 0; i < s.size(); ++i) t += (i ? "x" : "") + std::to_string(s[i]);
  return s.empty() ? "scalar" : t;
}

SppLevel spp_level(int64_t height, int64_t width, int level) {
  SppLevel v;
  v.bins = int64_t(1) << level;
  v.kernel_h = (height + v.bins - 1) / v.bins;  // ceil(bottom_h / double(num_bins)) for positive sizes
  v.kernel_w = (width + v.bins - 1) / v.bins;
  v.pad_h = (v.kernel_h * v.bins - height + 1) / 2;
  v.pad_w = (v.kernel_w * v.bins - width + 1) / 2;
  return v;
}

namespace {

typedef std::vector<int64_t> Shape;

std::string shape_string(const Shape& s) {  // Blob::shape_string: "2 3 4 (24)"
  std::string t;
  for (int64_t d : s) t += std::to_string(d) + " ";
  return t + "(" + std::to_string(shape_count(s)) + ")";
}

// ------------------------------------------------- protobuf text-format reader
struct Node {
  bool is_msg = false;
  std::string value;                                             // scalar
  std::vector<std::pair<std::string, std::shared_ptr<Node>>> kids;  // message fields, in order

  std::vector<const Node*> all(const std::string& key) const {
    std::vector<const Node*> out;
    for (const auto& kv : kids)
      if (kv.first == key) out.push_back(kv.second.get());
    return out;
  }
  const Node* first(const std::string& key) const {
    for (const auto& kv : kids)
      if (kv.first == key) return kv.second.get();
    return nullptr;
  }
  std::string str(const std::string& key, const std::string& dflt = "") const {
    const Node* n = first(key);
    return (n && !n->is_msg) ? n->value : dflt;
  }
  double num(const std::string& key, double dflt) const {
    const Node* n = first(key);
    return (n && !n->is_msg) ? atof(n->value.c_str()) : dflt;
  }
  long integer(const std::string& key, long dflt) const {
    const Node* n = first(key);
    return (n && !n->is_msg) ? atol(n->value.c_str()) : dflt;
  }
  bool boolean(const std::string& key, bool dflt) const {
    const Node* n = first(key);
    if (!n || n->is_msg) return dflt;
    return n->value == "true" || n->value == "1" || n->value == "True";
  }
};

class TextParser {
 public:
  explicit TextParser(const std::string& s) : s_(s) {}
  bool parse(Node* root, std::string* err) {
    root->is_msg = true;
    if (!message(root, /*top=*/true)) {
      std::ostringstream os;
      os << "prototxt parse error near offset " << pos_ << ": " << err_;
      *err = os.str();
      return false;
    }
    return true;
  }

 private:
  void skip() {
    for (;;) {
      while (pos_ < s_.size() && (isspace(static_cast<unsigned char>(s_[pos_])) || s_[pos_] == ',' || s_[pos_] == ';'))
        ++pos_;
      if (pos_ < s_.size() && s_[pos_] == '#') {
        while (pos_ < s_.size() && s_[pos_] != '\n') ++pos_;
        continue;
      }
      break;
    }
  }
  bool word(std::string* out) {
    skip();
    size_t b = pos_;
    while (pos_ < s_.size()) {
      char c = s_[pos_];
      if (isalnum(static_cast<unsigned char>(c)) || c == '_' || c == '.' || c == '+' || c == '-') ++pos_;
      else break;
    }
    if (pos_ == b) return false;
    *out = s_.substr(b, pos_ - b);
    return true;
  }
  bool quoted(std::string* out) {
    skip();
    if (pos_ >= s_.size() || (s_[pos_] != '"' && s_[pos_] != '\'')) return false;
    out->clear();
    while (pos_ < s_.size() && (s_[pos_] == '"' || s_[pos_] == '\'')) {  // adjacent strings concatenate
      char q = s_[pos_++];
      while (pos_ < s_.size() && s_[pos_] != q) {
        if (s_[pos_] == '\\' && pos_ + 1 < s_.size()) {
          char e = s_[pos_ + 1];
          out->push_back(e == 'n' ? '\n' : e == 't' ? '\t' : e);
          pos_ += 2;
        } else {
          out->push_back(s_[pos_++]);
        }
      }
      if (pos_ >= s_.size()) { err_ = "unterminated string"; return false; }
      ++pos_;
      skip();
    }
    return true;
  }
  bool message(Node* m, bool top) {
    for (;;) {
      skip();
      if (pos_ >= s_.size()) {
        if (top) return true;
        err_ = "missing '}'";
        return false;
      }
      if (s_[pos_] == '}' || s_[pos_] == '>') {
        if (top) { err_ = "unexpected '}'"; return false; }
        ++pos_;
        return true;
      }
      std::string key;
      if (!word(&key)) { err_ = "expected field name"; return false; }
      skip();
      bool colon = false;
      if (pos_ < s_.size() && s_[pos_] == ':') { colon = true; ++pos_; skip(); }
      auto child = std::make_shared<Node>();
      if (pos_ < s_.size() && (s_[pos_] == '{' || s_[pos_] == '<')) {
        ++pos_;
        child->is_msg = true;
        if (!message(child.get(), false)) return false;
      } else if (colon) {
        if (pos_ < s_.size() && s_[pos_] == '[') {  // short repeated form: [a, b]
          ++pos_;
          for (;;) {
            skip();
            if (pos_ < s_.size() && s_[pos_] == ']') { ++pos_; break; }
            auto item = std::make_shared<Node>();
            if (!quoted(&item->value) && !word(&item->value)) { err_ = "bad list item"; return false; }
            m->kids.emplace_back(key, item);
          }
          continue;
        }
        if (!quoted(&child->value) && !word(&child->value)) { err_ = "expected value for '" + key + "'"; return false; }
      } else {
        err_ = "expected ':' or '{' after '" + key + "'";
        return false;
      }
      m->kids.emplace_back(key, child);
    }
  }
  const std::string& s_;
  size_t pos_ = 0;
  std::string err_;
};

bool read_file(const std::string& path, std::string* out) {
  std::ifstream f(path.c_str(), std::ios::in | std::ios::binary);
  if (!f) return false;
  std::ostringstream ss;
  ss << f.rdbuf();
  *out = ss.str();
  return true;
}

// NetStateRule filtering for phase TRAIN (net.cpp FilterNet/StateMeetsRule;
// only the phase criterion is modelled).
bool in_train_phase(const Node& layer) {
  auto includes = layer.all("include");
  auto excludes = layer.all("exclude");
  if (!includes.empty()) {
    for (const Node* r : includes) {
      std::string ph = r->str("phase");
      if (ph.empty() || ph == "TRAIN") return true;
    }
    return false;
  }
  for (const Node* r : excludes) {
    std::string ph = r->str("phase");
    if (ph.empty() || ph == "TRAIN") return false;
  }
  std::string own = layer.str("phase");  // rarely used layer-level phase
  return own.empty() || own == "TRAIN";
}

struct HW { int64_t h, w; };

// kernel_size / kernel_h,kernel_w style repeated-or-pair fields
HW pair_field(const Node& p, const std::string& rep, const std::string& h, const std::string& w, int64_t dflt) {
  HW r{dflt, dflt};
  auto reps = p.all(rep);
  if (reps.size() == 1) r.h = r.w = atol(reps[0]->value.c_str());
  else if (reps.size() >= 2) { r.h = atol(reps[0]->value.c_str()); r.w = atol(reps[1]->value.c_str()); }
  if (p.first(h)) r.h = p.integer(h, dflt);
  if (p.first(w)) r.w = p.integer(w, dflt);
  return r;
}

FillerSpec filler(const Node* f) {
  FillerSpec s;
  if (!f || !f->is_msg) return s;
  s.type = f->str("type", "constant");
  s.value = static_cast<float>(f->num("value", 0.0));
  s.min = static_cast<float>(f->num("min", 0.0));
  s.max = static_cast<float>(f->num("max", 1.0));
  s.mean = static_cast<float>(f->num("mean", 0.0));
  s.std = static_cast<float>(f->num("std", 1.0));
  s.variance_norm = f->str("variance_norm", "FAN_IN");
  s.sparse = f->integer("sparse", -1);
  return s;
}

// TransformationParameter; force_color / force_gray only matter for decoding, which happens before the library.
TransformSpec transform(const Node* t, const std::string& net_file) {
  TransformSpec s;
  if (!t || !t->is_msg) return s;
  s.present = true;
  s.scale = static_cast<float>(t->num("scale", 1.0));
  s.mirror = t->boolean("mirror", false);
  s.crop_size = t->integer("crop_size", 0);
  s.mean_file = t->str("mean_file", "");
  s.net_file = net_file;
  for (const Node* v : t->all("mean_value")) s.mean_values.push_back(static_cast<float>(atof(v->value.c_str())));
  return s;
}

// What a rule works with: `rec` arrives with the common fields set; spec, net_file and first_data serve data layers.
struct Layer {
  const Node& node;
  NetLayer& rec;
  std::map<std::string, Shape>& blobs;  // every blob so far, by name
  std::string* err;
  SolverSpec* spec;
  const std::string& net_file;
  bool& first_data;  // no data layer has given the net its batch_size and input_shape yet
  bool bottom(size_t i, Shape* s) const {
    if (i >= rec.bottoms.size() || !blobs.count(rec.bottoms[i])) return refuse("unknown bottom blob");
    *s = blobs.at(rec.bottoms[i]);
    return true;
  }
  void set_top(size_t i, const Shape& s) { if (i < rec.tops.size()) blobs[rec.tops[i]] = s; }
  void set_tops(const Shape& s) { for (const std::string& t : rec.tops) blobs[t] = s; }
  bool refuse(const std::string& reason) const { *err = "layer '" + rec.name + "' (" + rec.type + "): " + reason; return false; }
  // the older wording, without the type ("layer 'c': bad Convolution"); an unknown bottom reported first stands
  bool bad(const std::string& what) const { if (err->empty()) *err = "layer '" + rec.name + "': bad " + what; return false; }
};

// A rule infers the layer's top shapes, refuses what Caffe would refuse, and appends the shapes of the learnable blobs
// the layer owns to `params`, in Caffe's order.
typedef bool (*Rule)(Layer& L, std::vector<Shape>* params);

bool canonical_axis(const Layer& L, int64_t given, int64_t naxes, int64_t* axis) {  // Blob::CanonicalAxisIndex
  *axis = given < 0 ? given + naxes : given;
  if (*axis < 0 || *axis >= naxes)
    return L.refuse("axis " + std::to_string(given) + " out of range for " + std::to_string(naxes) + "-D Blob");
  return true;
}

// Top i of a data layer, of shape s, as a staged input with `transform_param`.
void data_top(Layer& L, size_t i, Shape s, const Node* transform_param) {
  L.set_top(i, s);
  StagedInput in;
  in.layer = L.rec.name, in.type = L.rec.type, in.top = L.rec.tops[i], in.shape = s;
  in.transform = transform(transform_param, L.net_file);
  L.spec->inputs.push_back(in);
}

// The first data layer to call it gives the net's batch and input shape; the batch is s[0] unless given (a transposed
// CoSData top is [channels, batch_size]).
void data_input(Layer& L, const Shape& s, int64_t batch = -1) {
  if (!L.first_data) return;
  L.spec->batch_size = static_cast<int>(batch >= 0 ? batch : s[0]);
  L.spec->input_shape.assign(s.begin(), s.end());
  L.first_data = false;
}

bool memory_data(Layer& L, std::vector<Shape>*) {
  const Node* p = L.node.first("memory_data_param");
  if (!p) { *L.err = "MemoryData layer without memory_data_param"; return false; }
  Shape s{p->integer("batch_size", 0), p->integer("channels", 0), p->integer("height", 0), p->integer("width", 0)};
  L.set_top(0, s), L.set_top(1, Shape{s[0]});  // data and label, both set before a top is staged with its name's shape
  for (size_t i = 0; i < L.rec.tops.size(); ++i)  // the transform applies to the data, never to the label
    data_top(L, i, L.blobs[L.rec.tops[i]], i == 0 ? L.node.first("transform_param") : nullptr);
  data_input(L, s);  // even without a top
  return true;
}

bool cos_data(Layer& L, std::vector<Shape>*) {
  const Node* p = L.node.first("cos_data_param");
  if (!p) { *L.err = "CoSData layer without cos_data_param"; return false; }
  auto tb = p->all("top");
  const int64_t batch = p->integer("batch_size", 0);
  for (size_t i = 0; i < L.rec.tops.size(); ++i) {
    Shape s{batch};
    if (i < tb.size()) {
      int64_t c = tb[i]->integer("out_channels", 0), h = tb[i]->integer("out_height", 0), w = tb[i]->integer("out_width", 0);
      if (!c) c = tb[i]->integer("channels", 0);
      if (!h) h = tb[i]->integer("height", 0);
      if (!w) w = tb[i]->integer("width", 0);
      const int64_t axes = tb[i]->integer("sample_num_axes", 3);
      if (tb[i]->boolean("transpose", false)) {  // cos_data_layer.cpp: time-major [channels, batch_size]
        if (axes != 1) return L.refuse("each sample must be a 1d-vector if transpose is used");
        s = {c, batch};
      } else {
        Shape full{c, h, w};
        for (int64_t a = 0; a < axes && a < 3; ++a) s.push_back(full[a] ? full[a] : 1);
      }
    }
    data_top(L, i, s, i < tb.size() ? tb[i]->first("transform_param") : nullptr);
    if (i == 0) data_input(L, s, batch);
  }
  return true;
}

bool input(Layer& L, std::vector<Shape>*) {
  const Node* p = L.node.first("input_param");
  auto shapes = p ? p->all("shape") : std::vector<const Node*>();
  for (size_t i = 0; i < L.rec.tops.size(); ++i) {
    Shape s;
    if (!shapes.empty()) for (const Node* d : shapes[std::min(i, shapes.size() - 1)]->all("dim")) s.push_back(atol(d->value.c_str()));
    data_top(L, i, s, nullptr);
    if (i == 0 && !s.empty()) data_input(L, s);
  }
  return true;
}

// base_conv_layer.cpp LayerSetUp's rule for a repeated field of an N-D convolution: given once, or once per spatial
// axis, or (with a default) not at all; the _h / _w form only in 2-D.  False, with Caffe's CHECK wording, otherwise.
// `hw` names the 2-D form's prefix ("" for dilation, which has none).
bool spatial_field(const Layer& L, const Node& p, const std::string& name, const std::string& hw, size_t axes,
                   int64_t dflt, std::vector<int64_t>* out) {
  if (!hw.empty() && (p.first(hw + "_h") || p.first(hw + "_w")))
    return L.refuse(hw + "_h & " + hw + "_w can only be used for 2D convolution.");
  auto reps = p.all(name);
  if (!(reps.size() == 1 || reps.size() == axes || (reps.empty() && dflt >= 0)))
    return L.refuse(name + " must be specified once, or once per spatial dimension (" + name + " specified " +
                    std::to_string(reps.size()) + " times; " + std::to_string(axes) + " spatial dims).");
  out->assign(axes, dflt);
  for (size_t a = 0; a < axes && !reps.empty(); ++a) (*out)[a] = atol(reps[reps.size() == 1 ? 0 : a]->value.c_str());
  return true;
}

// A Convolution or Deconvolution over a bottom of 3 or 5 axes, [N, C, L] or [N, C, D, H, W]: base_conv_layer.cpp's
// per-axis fields and conv_layer.cpp / deconv_layer.cpp's output size on every spatial axis.  A 1-D layer is recorded
// as the 2-D one over [N, C, 1, L] (kernel_h 1, stride_h 1, pad_h 0); a 3-D layer adds the depth fields.
bool convolution_nd(Layer& L, const Node& p, const Shape& in, std::vector<Shape>* params) {
  int64_t axis = 0;
  if (!canonical_axis(L, p.integer("axis", 1), static_cast<int64_t>(in.size()), &axis)) return false;
  if (axis != 1)
    return L.refuse("convolution_param axis " + std::to_string(p.integer("axis", 1)) + " is not supported on a " +
                    std::to_string(in.size()) + "-axis bottom (the channel axis must be 1)");
  const size_t axes = in.size() - 2;
  std::vector<int64_t> k, st, pad, dil;
  if (!spatial_field(L, p, "kernel_size", "kernel", axes, -1, &k)) return false;
  for (int64_t v : k)
    if (v <= 0) return L.refuse("Filter dimensions must be nonzero.");
  if (!spatial_field(L, p, "stride", "stride", axes, 1, &st)) return false;
  for (int64_t v : st)
    if (v <= 0) return L.refuse("Stride dimensions must be nonzero.");
  if (!spatial_field(L, p, "pad", "pad", axes, 0, &pad) || !spatial_field(L, p, "dilation", "", axes, 1, &dil))
    return false;
  const int64_t nout = p.integer("num_output", 0), group = p.integer("group", 1);
  bool ok = nout > 0 && group > 0 && in[1] % group == 0 && nout % group == 0;
  for (size_t a = 0; a < axes; ++a) ok = ok && pad[a] >= 0 && dil[a] > 0;
  if (!ok) return L.bad("convolution_param");
  NetLayer& r = L.rec;
  r.num_output = nout, r.group = group;
  const size_t h = axes == 3 ? 1 : 0, w = axes - 1;  // the height and width axes among the spatial ones (1-D: H = 1)
  if (axes == 3) r.kernel_d = k[0], r.stride_d = st[0], r.pad_d = pad[0], r.dilation_d = dil[0];
  r.kernel_h = axes == 1 ? 1 : k[h], r.stride_h = axes == 1 ? 1 : st[h], r.pad_h = axes == 1 ? 0 : pad[h];
  r.dilation_h = axes == 1 ? 1 : dil[h];
  r.kernel_w = k[w], r.stride_w = st[w], r.pad_w = pad[w], r.dilation_w = dil[w];
  r.bias_term = p.boolean("bias_term", true);
  r.weight_filler = filler(p.first("weight_filler")), r.bias_filler = filler(p.first("bias_filler"));
  const bool conv = r.type == "Convolution";
  Shape weight{conv ? nout : in[1], conv ? in[1] / group : nout / group}, top{in[0], nout};
  for (size_t a = 0; a < axes; ++a) {
    const int64_t ke = dil[a] * (k[a] - 1) + 1;  // the dilated kernel
    weight.push_back(k[a]);
    top.push_back(conv ? (in[2 + a] + 2 * pad[a] - ke) / st[a] + 1 : st[a] * (in[2 + a] - 1) + ke - 2 * pad[a]);
  }
  params->push_back(weight);
  L.set_top(0, top);
  if (r.bias_term) params->push_back({nout});
  return true;
}

bool convolution(Layer& L, std::vector<Shape>* params) {  // and Deconvolution; weight shapes of base_conv_layer.cpp
  const Node* p = L.node.first("convolution_param");
  Shape in;
  if (p && L.bottom(0, &in) && in.size() >= 6)
    return L.refuse("a bottom of " + std::to_string(in.size()) + " axes is not supported (at most 3 spatial axes are)");
  if (p && (in.size() == 3 || in.size() == 5)) return convolution_nd(L, *p, in, params);
  if (!p || !L.bottom(0, &in) || in.size() != 4) return L.bad("Convolution");
  const int64_t nout = p->integer("num_output", 0), group = p->integer("group", 1);
  HW k = pair_field(*p, "kernel_size", "kernel_h", "kernel_w", 0), st = pair_field(*p, "stride", "stride_h", "stride_w", 1);
  HW pad = pair_field(*p, "pad", "pad_h", "pad_w", 0), dil = pair_field(*p, "dilation", "dilation_h", "dilation_w", 1);
  if (nout <= 0 || k.h <= 0 || k.w <= 0 || group <= 0 || in[1] % group || nout % group || st.h <= 0 || st.w <= 0 ||
      dil.h <= 0 || dil.w <= 0 || pad.h < 0 || pad.w < 0)
    return L.bad("convolution_param");
  NetLayer& r = L.rec;
  r.num_output = nout, r.group = group;
  r.kernel_h = k.h, r.kernel_w = k.w, r.stride_h = st.h, r.stride_w = st.w;
  r.pad_h = pad.h, r.pad_w = pad.w, r.dilation_h = dil.h, r.dilation_w = dil.w;
  r.bias_term = p->boolean("bias_term", true);
  r.weight_filler = filler(p->first("weight_filler")), r.bias_filler = filler(p->first("bias_filler"));
  const int64_t kh = dil.h * (k.h - 1) + 1, kw = dil.w * (k.w - 1) + 1;  // the dilated kernel
  if (r.type == "Convolution") {
    params->push_back({nout, in[1] / group, k.h, k.w});
    L.set_top(0, {in[0], nout, (in[2] + 2 * pad.h - kh) / st.h + 1, (in[3] + 2 * pad.w - kw) / st.w + 1});
  } else {
    params->push_back({in[1], nout / group, k.h, k.w});
    L.set_top(0, {in[0], nout, st.h * (in[2] - 1) + kh - 2 * pad.h, st.w * (in[3] - 1) + kw - 2 * pad.w});
  }
  if (r.bias_term) params->push_back({nout});
  return true;
}

// pooling_layer.cpp's pad < kernel CHECKs (LayerSetUp), with `at` after their wording, and its pooled size (Reshape)
bool pooled(const Layer& L, HW in, HW k, HW st, HW pad, const std::string& at, HW* out) {
  // a window that lay entirely in the padding would pool nothing
  if (pad.h >= k.h)
    return L.refuse("Check failed: pad_h_ < kernel_h_ (" + std::to_string(pad.h) + " vs. " + std::to_string(k.h) + ")" +
                    at);
  if (pad.w >= k.w)
    return L.refuse("Check failed: pad_w_ < kernel_w_ (" + std::to_string(pad.w) + " vs. " + std::to_string(k.w) + ")" +
                    at);
  // ceil((H + 2p - k) / s) + 1, clipped so the last window starts inside
  out->h = static_cast<int64_t>(ceil(static_cast<float>(in.h + 2 * pad.h - k.h) / st.h)) + 1;
  out->w = static_cast<int64_t>(ceil(static_cast<float>(in.w + 2 * pad.w - k.w) / st.w)) + 1;
  if (pad.h || pad.w) {
    if ((out->h - 1) * st.h >= in.h + pad.h) --out->h;
    if ((out->w - 1) * st.w >= in.w + pad.w) --out->w;
  }
  return true;
}

bool pooling(Layer& L, std::vector<Shape>*) {
  const Node* p = L.node.first("pooling_param");
  Shape in;
  if (!p || !L.bottom(0, &in) || in.size() != 4) return L.bad("Pooling");
  HW k = pair_field(*p, "kernel_size", "kernel_h", "kernel_w", 0), st = pair_field(*p, "stride", "stride_h", "stride_w", 1);
  HW pad = pair_field(*p, "pad", "pad_h", "pad_w", 0);
  const bool global = p->boolean("global_pooling", false);
  if (global) {  // pooling_layer.cpp LayerSetUp's checks, in its order
    if (p->first("kernel_size") || p->first("kernel_h") || p->first("kernel_w"))
      return L.refuse("With Global_pooling: true Filter size cannot specified");
    k.h = in[2], k.w = in[3];
  }
  if (k.h <= 0 || k.w <= 0 || st.h <= 0 || st.w <= 0 || pad.h < 0 || pad.w < 0) return L.bad("pooling_param");
  if (global && (pad.h || pad.w || st.h != 1 || st.w != 1))
    return L.refuse("With Global_pooling: true; only pad = 0 and stride = 1");
  HW out;
  if (!pooled(L, {in[2], in[3]}, k, st, pad, "", &out)) return false;
  NetLayer& r = L.rec;
  r.kernel_h = k.h, r.kernel_w = k.w, r.stride_h = st.h, r.stride_w = st.w, r.pad_h = pad.h, r.pad_w = pad.w;
  r.pool = p->str("pool", "MAX"), r.global_pooling = global;
  L.set_tops({in[0], in[1], out.h, out.w});
  return true;
}

// spp_layer.cpp: Reshape's CHECK, LayerSetUp's, then each level's Pooling (GetPoolingParam, spp_level) through
// pooled().  One level is Caffe's lone Pooling with its [N, C, 1, 1] top; more are the Concat of each level's
// Flatten, [N, C * sum of bins^2].
bool spp(Layer& L, std::vector<Shape>*) {
  Shape in;
  if (!L.bottom(0, &in)) return false;
  if (in.size() != 4) return L.refuse("Input must have 4 axes, corresponding to (num, channels, height, width)");
  if (in[2] <= 0 || in[3] <= 0) return L.refuse("Input dimensions cannot be zero.");
  const Node* p = L.node.first("spp_param");
  NetLayer& r = L.rec;
  r.pyramid_height = p ? p->integer("pyramid_height", 0) : 0;
  if (r.pyramid_height < 1)
    return L.refuse("spp_param pyramid_height must be at least 1 (a pyramid of no levels pools nothing)");
  r.pool = p->str("pool", "MAX");
  int64_t per_channel = 0;
  for (int l = 0; l < r.pyramid_height; ++l) {
    const SppLevel v = spp_level(in[2], in[3], l);
    HW out;
    const std::string at = " at pyramid level " + std::to_string(l) + " (" + std::to_string(v.bins) + " bins)";
    if (!pooled(L, {in[2], in[3]}, {v.kernel_h, v.kernel_w}, {v.kernel_h, v.kernel_w}, {v.pad_h, v.pad_w}, at, &out))
      return false;
    per_channel += out.h * out.w;
  }
  L.set_top(0, r.pyramid_height == 1 ? Shape{in[0], in[1], 1, 1} : Shape{in[0], in[1] * per_channel});
  return true;
}

bool inner_product(Layer& L, std::vector<Shape>* params) {
  const Node* p = L.node.first("inner_product_param");
  Shape in;
  if (!p || !L.bottom(0, &in)) return L.bad("InnerProduct");
  const int64_t nout = p->integer("num_output", 0), naxes = static_cast<int64_t>(in.size());
  int64_t axis = p->integer("axis", 1);
  if (axis < 0) axis += naxes;
  if (nout <= 0 || axis < 0 || axis > naxes) return L.bad("inner_product_param");
  NetLayer& r = L.rec;
  r.num_output = nout, r.axis = axis;
  r.bias_term = p->boolean("bias_term", true), r.transpose = p->boolean("transpose", false);
  r.weight_filler = filler(p->first("weight_filler")), r.bias_filler = filler(p->first("bias_filler"));
  params->push_back({nout, shape_count(in, static_cast<size_t>(axis))});  // inner_product_layer.cpp: N x K
  if (r.bias_term) params->push_back({nout});
  Shape out(in.begin(), in.begin() + axis);
  out.push_back(nout);
  L.set_top(0, out);
  return true;
}

bool same_shape(Layer& L, std::vector<Shape>*) {  // ReLU, LRN, Dropout, Sigmoid, ...
  Shape in;
  if (!L.bottom(0, &in)) return false;
  L.set_tops(in);
  NetLayer& r = L.rec;
  if (const Node* p = L.node.first("relu_param")) r.negative_slope = static_cast<float>(p->num("negative_slope", 0.0));
  if (const Node* p = L.node.first("lrn_param")) {  // caffe.proto LRNParameter
    r.local_size = p->integer("local_size", 5);
    r.lrn_alpha = static_cast<float>(p->num("alpha", 1.0));
    r.lrn_beta = static_cast<float>(p->num("beta", 0.75));
    r.lrn_k = static_cast<float>(p->num("k", 1.0));
    r.norm_region = p->str("norm_region", "ACROSS_CHANNELS");
    if (r.norm_region == "0") r.norm_region = "ACROSS_CHANNELS";  // the enum's numeric form
    if (r.norm_region == "1") r.norm_region = "WITHIN_CHANNEL";
  }
  // the neuron layers' parameters with caffe.proto's defaults; the engine's plan checks them
  if (const Node* p = L.node.first("power_param")) {
    r.power = static_cast<float>(p->num("power", 1.0));
    r.scale = static_cast<float>(p->num("scale", 1.0));
    r.shift = static_cast<float>(p->num("shift", 0.0));
  }
  const Node* exp_log = r.type == "Exp" ? L.node.first("exp_param") : r.type == "Log" ? L.node.first("log_param") : nullptr;
  if (exp_log) {
    r.base = static_cast<float>(exp_log->num("base", -1.0));
    r.scale = static_cast<float>(exp_log->num("scale", 1.0));
    r.shift = static_cast<float>(exp_log->num("shift", 0.0));
  }
  if (const Node* p = L.node.first("elu_param")) r.elu_alpha = static_cast<float>(p->num("alpha", 1.0));
  if (const Node* p = L.node.first("threshold_param")) r.threshold = static_cast<float>(p->num("threshold", 0.0));
  if (const Node* p = L.node.first("softmax_param")) r.softmax_axis = p->integer("axis", 1);
  return true;
}

bool prelu(Layer& L, std::vector<Shape>* params) {  // prelu_layer.cpp LayerSetUp: one slope per channel, or a scalar
  Shape in;
  if (!L.bottom(0, &in)) return false;
  const Node* p = L.node.first("prelu_param");
  NetLayer& r = L.rec;
  r.channel_shared = p && p->boolean("channel_shared", false);
  if (p && p->first("filler")) r.weight_filler = filler(p->first("filler"));
  else r.weight_filler.value = 0.25f;  // Caffe's default: constant 0.25
  // Blob::channels() of a bottom with fewer than 2 axes is 1; the engine refuses such a bottom with Caffe's wording
  params->push_back(r.channel_shared ? Shape{} : Shape{in.size() >= 2 ? in[1] : 1});
  L.set_tops(in);
  return true;
}

bool split(Layer& L, std::vector<Shape>*) {  // split_layer.cpp Reshape
  Shape in;
  if (!L.bottom(0, &in)) return false;
  for (const std::string& t : L.rec.tops) {
    if (t == L.rec.bottoms[0]) return L.refuse("Split Layer does not allow in-place computation.");
    L.blobs[t] = in;
  }
  return true;
}

bool eltwise(Layer& L, std::vector<Shape>*) {  // eltwise_layer.cpp LayerSetUp and Reshape, after Layer::CheckBlobCounts
  const size_t n = L.rec.bottoms.size();
  if (n < 2) return L.refuse("Eltwise Layer takes at least 2 bottom blob(s) as input.");
  Shape in;
  if (!L.bottom(0, &in)) return false;
  const Node* p = L.node.first("eltwise_param");
  auto coeffs = p ? p->all("coeff") : std::vector<const Node*>();
  if (!coeffs.empty() && coeffs.size() != n) return L.refuse("Eltwise Layer takes one coefficient per bottom blob.");
  std::string op = p ? p->str("operation", "SUM") : "SUM";
  if (op == "0") op = "PROD";  // the enum's numeric form
  if (op == "1") op = "SUM";
  if (op == "2") op = "MAX";
  if (op != "PROD" && op != "SUM" && op != "MAX") return L.refuse("Unknown elementwise operation.");
  if (op == "PROD" && !coeffs.empty()) return L.refuse("Eltwise layer only takes coefficients for summation.");
  L.rec.eltwise_op = op, L.rec.coeffs.assign(n, 1.f);
  for (size_t i = 0; i < coeffs.size(); ++i) L.rec.coeffs[i] = static_cast<float>(atof(coeffs[i]->value.c_str()));
  L.rec.stable_prod_grad = !p || p->boolean("stable_prod_grad", true);
  for (size_t i = 1; i < n; ++i) {
    Shape s;
    if (!L.bottom(i, &s)) return false;
    if (s != in)
      return L.refuse("bottom " + std::to_string(i) + " is " + shape_text(s) + ", bottom 0 " + shape_text(in) +
                      " (Check failed: bottom[i]->shape() == bottom[0]->shape())");
  }
  L.set_tops(in);
  return true;
}

bool scale(Layer& L, std::vector<Shape>* params) {  // scale_layer.cpp LayerSetUp and Reshape; the bias as bias_layer.cpp
  if (L.rec.bottoms.size() > 2) return L.refuse("Scale Layer takes at most 2 bottom blob(s) as input.");
  Shape in;
  if (!L.bottom(0, &in)) return false;
  const Node* p = L.node.first("scale_param");
  const int64_t naxes = static_cast<int64_t>(in.size());
  int64_t axis;
  if (!canonical_axis(L, p ? p->integer("axis", 1) : 1, naxes, &axis)) return false;
  const std::string past = "scale blob's shape extends past bottom[0]'s shape when applied starting with bottom[0] axis = ";
  Shape scale;  // the scale blob's shape, or bottom[1]'s
  if (L.rec.bottoms.size() == 1) {
    const int64_t num_axes = p ? p->integer("num_axes", 1) : 1;
    if (num_axes < -1) return L.refuse("num_axes must be non-negative, or -1 to extend to the end of bottom[0]");
    if (num_axes >= 0 && naxes < axis + num_axes) return L.refuse(past + std::to_string(axis));
    scale.assign(in.begin() + axis, num_axes == -1 ? in.end() : in.begin() + axis + num_axes);
    params->push_back(scale);
  } else if (!L.bottom(1, &scale)) {
    return false;
  }
  const int64_t first = scale.empty() ? 0 : axis;  // Reshape: a scalar scale applies from axis 0
  if (naxes < first + static_cast<int64_t>(scale.size())) return L.refuse(past + std::to_string(first));
  for (size_t i = 0; i < scale.size(); ++i)
    if (in[first + i] != scale[i])
      return L.refuse("dimension mismatch between bottom[0]->shape(" + std::to_string(first + i) + ") and scale->shape(" +
                      std::to_string(i) + ")");
  NetLayer& r = L.rec;
  r.bias_term = p && p->boolean("bias_term", false);
  if (r.bias_term) params->push_back(scale);  // the Bias layer's blob, of the scale's (or bottom[1]'s) shape
  r.axis = first, r.num_axes = static_cast<int64_t>(scale.size());
  if (p && p->first("filler")) r.weight_filler = filler(p->first("filler"));
  else r.weight_filler.value = 1.f;  // unit scale: a constant 1 filler
  r.bias_filler = filler(p ? p->first("bias_filler") : nullptr);
  L.set_tops(in);
  return true;
}

bool flatten(Layer& L, std::vector<Shape>*) {  // flatten_layer.cpp with its default axis 1 and end_axis -1
  Shape in;
  int64_t axis;  // CanonicalAxisIndex(1) refuses a 0-axis bottom; a 1-axis one, which Caffe refuses too, gives N x 1
  if (!L.bottom(0, &in) || (in.empty() && !canonical_axis(L, 1, 0, &axis))) return false;
  if (const Node* p = L.node.first("flatten_param")) {  // recorded for the engine, which runs the default alone
    L.rec.flatten_axis = p->integer("axis", 1);
    L.rec.flatten_end_axis = p->integer("end_axis", -1);
  }
  L.set_top(0, {in[0], shape_count(in, 1)});
  return true;
}

// Ids reach the engine as fp32, which holds every integer exactly only up to 2^24
constexpr int64_t kMaxEmbedInputDim = int64_t(1) << 24;

bool embed(Layer& L, std::vector<Shape>* params) {  // embed_layer.cpp LayerSetUp and Reshape, with its CHECK messages
  Shape in;
  if (!L.bottom(0, &in)) return false;
  const Node* p = L.node.first("embed_param");
  NetLayer& r = L.rec;
  r.num_output = p ? p->integer("num_output", 0) : 0;
  r.input_dim = p ? p->integer("input_dim", 0) : 0;
  if (r.num_output <= 0) return L.refuse("EmbedLayer num_output must be positive.");
  if (r.input_dim <= 0) return L.refuse("EmbedLayer input_dim must be positive.");
  if (r.input_dim > kMaxEmbedInputDim)
    return L.refuse("input_dim " + std::to_string(r.input_dim) + " is more than 2^24 = " +
                    std::to_string(kMaxEmbedInputDim) + ": ids arrive as fp32, which is not exact above it");
  r.bias_term = !p || p->boolean("bias_term", true);
  r.weight_filler = filler(p ? p->first("weight_filler") : nullptr);
  r.bias_filler = filler(p ? p->first("bias_filler") : nullptr);
  params->push_back({r.input_dim, r.num_output});  // transposed from InnerProduct's: one row per id
  if (r.bias_term) params->push_back({r.num_output});
  Shape out = in;
  out.push_back(r.num_output);
  L.set_top(0, out);
  return true;
}

bool reshape(Layer& L, std::vector<Shape>*) {  // reshape_layer.cpp LayerSetUp and Reshape, with its CHECK messages
  Shape in;
  if (!L.bottom(0, &in)) return false;
  const Node* p = L.node.first("reshape_param");
  const Node* shape = p ? p->first("shape") : nullptr;
  Shape dims;
  if (shape) for (const Node* d : shape->all("dim")) dims.push_back(atol(d->value.c_str()));
  int64_t inferred = -1, constant = 1;
  std::vector<int64_t> copies;
  for (size_t i = 0; i < dims.size(); ++i) {
    if (dims[i] == 0) {
      copies.push_back(static_cast<int64_t>(i));
    } else if (dims[i] == -1) {
      if (inferred != -1)
        return L.refuse("new shape contains multiple -1 dims; at most a single (1) value of -1 may be specified");
      inferred = static_cast<int64_t>(i);
    } else if (dims[i] < 0) {  // Blob::Reshape
      return L.refuse("Check failed: shape[" + std::to_string(i) + "] >= 0 (" + std::to_string(dims[i]) + " vs. 0)");
    } else {
      constant *= dims[i];
    }
  }
  const int64_t naxes = static_cast<int64_t>(in.size());
  const int64_t given = p ? p->integer("axis", 0) : 0;
  const int64_t start = given >= 0 ? given : naxes + given + 1;
  if (start < 0) return L.refuse("axis " + std::to_string(given) + " out of range");
  if (start > naxes)
    return L.refuse("axis " + std::to_string(given) + " out of range for " + std::to_string(naxes) + "-D input blob");
  const int64_t num_axes = p ? p->integer("num_axes", -1) : -1;
  if (num_axes < -1) return L.refuse("num_axes must be >= 0, or -1 for all");
  const int64_t end = num_axes == -1 ? naxes : start + num_axes;
  if (end > naxes) return L.refuse("end_axis = axis + num_axes is out of range");
  Shape out(in.begin(), in.begin() + start);
  out.insert(out.end(), dims.begin(), dims.end());
  out.insert(out.end(), in.begin() + end, in.end());
  for (int64_t c : copies) {
    if (naxes <= start + c)
      return L.refuse("new shape contains a 0, but there was no corresponding bottom axis to copy");
    out[start + c] = in[start + c];
  }
  if (inferred >= 0) {
    int64_t explicit_count = constant * shape_count(Shape(in.begin(), in.begin() + start)) * shape_count(in, end);
    for (int64_t c : copies) explicit_count *= out[start + c];
    if (explicit_count == 0 || shape_count(in) % explicit_count != 0)
      return L.refuse("bottom count (" + std::to_string(shape_count(in)) + ") must be divisible by the product of the "
                      "specified dimensions (" + std::to_string(explicit_count) + ")");
    out[start + inferred] = shape_count(in) / explicit_count;
  }
  if (shape_count(out) != shape_count(in)) return L.refuse("output count must match input count");
  L.set_top(0, out);
  return true;
}

// recurrent_layer.cpp LayerSetUp (after Layer::CheckBlobCounts) and rnn_layer.cpp FillUnrolledNet, with their CHECK
// messages.  The learnable blobs are the unrolled net's, in the order of their first use there: W_xh [H, I], b_h [H],
// W_xh_static [H, S] (with x_static), W_hh [H, H], W_ho [H, H], b_o [H], with I = count(x, 2) and S = count(x_static, 1).
bool rnn(Layer& L, std::vector<Shape>* params) {
  const Node* p = L.node.first("recurrent_param");
  NetLayer& r = L.rec;
  r.num_output = p ? p->integer("num_output", 0) : 0;
  r.expose_hidden = p && p->boolean("expose_hidden", false);
  const size_t least = 2 + (r.expose_hidden ? 1 : 0), tops = 1 + (r.expose_hidden ? 1 : 0);
  const std::string type = r.type + " Layer ";
  if (r.bottoms.size() < least)
    return L.refuse(type + "takes at least " + std::to_string(least) + " bottom blob(s) as input.");
  if (r.bottoms.size() > least + 1)
    return L.refuse(type + "takes at most " + std::to_string(least + 1) + " bottom blob(s) as input.");
  if (r.tops.size() != tops) return L.refuse(type + "produces " + std::to_string(tops) + " top blob(s) as output.");
  Shape x, cont, xs;
  if (!L.bottom(0, &x) || !L.bottom(1, &cont)) return false;
  if (x.size() < 2) return L.refuse("bottom[0] must have at least 2 axes -- (#timesteps, #streams, ...)");
  if (cont.size() != 2) return L.refuse("bottom[1] must have exactly 2 axes -- (#timesteps, #streams)");
  auto eq = [&](const char* what, int64_t a, int64_t b) {
    return a == b || L.refuse(std::string("Check failed: ") + what + " (" + std::to_string(a) + " vs. " +
                              std::to_string(b) + ")");
  };
  if (!eq("T_ == bottom[1]->shape(0)", x[0], cont[0]) || !eq("N_ == bottom[1]->shape(1)", x[1], cont[1])) return false;
  r.static_input = r.bottoms.size() > least;
  if (r.static_input) {
    if (!L.bottom(2, &xs)) return false;
    if (xs.empty()) return L.refuse("Check failed: bottom[2]->num_axes() >= 1 (0 vs. 1)");
    if (!eq("N_ == bottom[2]->shape(0)", x[1], xs[0])) return false;
  }
  if (r.num_output <= 0) return L.refuse("num_output must be positive");
  const int64_t H = r.num_output;
  r.weight_filler = filler(p->first("weight_filler")), r.bias_filler = filler(p->first("bias_filler"));  // p: H > 0
  *params = {{H, shape_count(x, 2)}, {H}};
  r.bias_param = {false, true};
  if (r.static_input) params->push_back({H, shape_count(xs, 1)}), r.bias_param.push_back(false);
  params->insert(params->end(), {{H, H}, {H, H}, {H}});
  r.bias_param.insert(r.bias_param.end(), {false, false, true});
  L.set_top(0, {x[0], x[1], H});
  if (r.expose_hidden) L.set_top(1, {1, x[1], H});
  return true;
}

bool concat(Layer& L, std::vector<Shape>*) {  // concat_layer.cpp LayerSetUp and Reshape, with its CHECK messages
  Shape out;
  if (!L.bottom(0, &out)) return false;
  const Node* p = L.node.first("concat_param");
  const int64_t naxes = static_cast<int64_t>(out.size());
  int64_t axis = 1;
  if (p && p->first("axis") && p->first("concat_dim")) return L.refuse("Either axis or concat_dim should be specified; not both.");
  if (p && p->first("concat_dim")) {  // a uint32: never counted from the end
    axis = p->integer("concat_dim", 1);
    if (axis < 0 || axis >= naxes) return L.refuse("concat_dim out of range.");
  } else if (!canonical_axis(L, p ? p->integer("axis", 1) : 1, naxes, &axis)) {
    return false;
  }
  for (size_t i = 1; i < L.rec.bottoms.size(); ++i) {
    Shape s;
    if (!L.bottom(i, &s)) return false;
    if (s.size() != out.size()) return L.refuse("All inputs must have the same #axes.");
    for (int64_t j = 0; j < naxes; ++j)
      if (j != axis && s[j] != out[j]) return L.refuse("All inputs must have the same shape, except at concat_axis.");
    out[axis] += s[axis];
  }
  L.rec.axis = axis;
  L.set_top(0, out);
  return true;
}

bool batch_norm(Layer& L, std::vector<Shape>* params) {
  // batch_norm_layer.cpp:17-36: mean [C], variance [C], moving-average scale factor [1]; C = shape(1), or 1
  // for a 1-axis bottom.  The forward pass rewrites them; their lr_mult is whatever the prototxt says.
  Shape in;
  if (!L.bottom(0, &in)) return false;
  if (in.empty()) return L.bad("BatchNorm bottom");
  const int64_t C = in.size() == 1 ? 1 : in[1];
  *params = {{C}, {C}, {1}};
  L.set_tops(in);
  if (const Node* p = L.node.first("batch_norm_param")) {  // caffe.proto BatchNormParameter
    L.rec.use_global_stats = p->boolean("use_global_stats", false);
    L.rec.moving_average_fraction = static_cast<float>(p->num("moving_average_fraction", 0.999));
    L.rec.eps = static_cast<float>(p->num("eps", 1e-5));
  }
  return true;
}

// mvn_layer.cpp Reshape: the top is the bottom's legacy 4-D shape (num, channels, height, width), with Blob::LegacyShape's
// CHECK; a zero dimension would make Forward divide by a zero count, so it is refused too
bool mvn(Layer& L, std::vector<Shape>*) {
  Shape in;
  if (!L.bottom(0, &in)) return false;
  if (in.size() > 4) return L.refuse("Cannot use legacy accessors on Blobs with > 4 axes.");
  Shape top(4, 1);
  for (size_t a = 0; a < in.size(); ++a) {
    if (in[a] == 0) return L.refuse("a bottom of shape " + shape_text(in) + " has no elements to normalise");
    top[a] = in[a];
  }
  L.set_tops(top);
  NetLayer& r = L.rec;
  r.eps = 1e-9f;
  if (const Node* p = L.node.first("mvn_param")) {
    r.normalize_variance = p->boolean("normalize_variance", true);
    r.across_channels = p->boolean("across_channels", false);
    r.eps = static_cast<float>(p->num("eps", 1e-9));
  }
  return true;
}

// crop_layer.cpp LayerSetUp and Reshape (after Layer::CheckBlobCounts), with their CHECK messages: bottom[0] cropped to
// bottom[1]'s size on every axis from `axis` on, at per-axis offsets.  bottom[1] gives only its shape.
bool crop(Layer& L, std::vector<Shape>*) {
  NetLayer& r = L.rec;
  if (r.bottoms.size() != 2) return L.refuse("Crop Layer takes 2 bottom blob(s) as input.");
  if (r.tops.size() != 1) return L.refuse("Crop Layer produces 1 top blob(s) as output.");
  const Node* p = L.node.first("crop_param");
  std::vector<int64_t> given;  // crop_param offset, a repeated uint32
  for (const Node* o : p ? p->all("offset") : std::vector<const Node*>()) {
    given.push_back(atol(o->value.c_str()));
    if (given.back() < 0) return L.refuse("crop_param offset " + o->value + ": Expected integer, got: -");
  }
  Shape in, ref;
  if (!L.bottom(0, &in) || !L.bottom(1, &ref)) return false;
  if (r.tops[0] == r.bottoms[0]) return L.refuse("Crop Layer does not allow in-place computation.");
  const int64_t naxes = static_cast<int64_t>(in.size());
  int64_t axis;
  if (!canonical_axis(L, p ? p->integer("axis", 2) : 2, naxes, &axis)) return false;
  if (given.size() > 1 && axis + static_cast<int64_t>(given.size()) != naxes)
    return L.refuse("number of offset values specified must be equal to the number of dimensions following axis.");
  Shape top = in;
  r.crop_offsets.assign(in.size(), 0);
  for (int64_t i = axis; i < naxes; ++i) {
    int64_t i_ref;  // Blob::shape(i) of the reference: CanonicalAxisIndex's CHECK
    if (!canonical_axis(L, i, static_cast<int64_t>(ref.size()), &i_ref)) return false;
    const int64_t offset = given.empty() ? 0 : given.size() == 1 ? given[0] : given[i - axis];
    if (in[i] - offset < ref[i])
      return L.refuse("the crop for dimension " + std::to_string(i) + " is out-of-bounds with size " +
                      std::to_string(ref[i]) + " and offset " + std::to_string(offset));
    top[i] = ref[i];
    r.crop_offsets[i] = offset;
  }
  r.axis = axis;
  L.set_top(0, top);
  return true;
}

// tile_layer.cpp Reshape, with its CHECK messages: the top is the bottom with shape[axis] *= tiles (axis default 1)
bool tile(Layer& L, std::vector<Shape>*) {
  Shape in;
  if (!L.bottom(0, &in)) return false;
  const Node* p = L.node.first("tile_param");
  NetLayer& r = L.rec;
  if (!canonical_axis(L, p ? p->integer("axis", 1) : 1, static_cast<int64_t>(in.size()), &r.axis)) return false;
  if (!p || !p->first("tiles")) return L.refuse("Number of tiles must be specified");
  r.tiles = p->integer("tiles", 0);
  if (r.tiles <= 0) return L.refuse("Number of tiles must be positive.");
  Shape top = in;
  top[r.axis] *= r.tiles;
  L.set_top(0, top);
  return true;
}

bool slice(Layer& L, std::vector<Shape>*) {  // slice_layer.cpp Reshape
  Shape in;
  if (!L.bottom(0, &in)) return false;
  const Node* p = L.node.first("slice_param");
  const int64_t naxes = static_cast<int64_t>(in.size());
  if (p && p->first("axis") && p->first("slice_dim")) return L.refuse("either axis or slice_dim should be specified; not both");
  const bool dim = p && p->first("slice_dim");  // slice_dim is never counted from the end
  int64_t axis = dim ? p->integer("slice_dim", 1) : p ? p->integer("axis", 1) : 1;
  if (!dim && axis < 0) axis += naxes;
  if (axis < 0 || axis >= naxes)
    return L.refuse("slice axis " + std::to_string(axis) + " is out of range for a " + std::to_string(naxes) + "-axis bottom");
  if (L.rec.tops.empty()) return L.refuse("needs at least one top");
  const int64_t A = in[axis], ntop = static_cast<int64_t>(L.rec.tops.size());
  std::vector<int64_t> bounds{0};
  auto points = p ? p->all("slice_point") : std::vector<const Node*>();
  if (!points.empty()) {
    if (static_cast<int64_t>(points.size()) != ntop - 1)
      return L.refuse(std::to_string(points.size()) + " slice_point(s) for " + std::to_string(ntop) + " tops");
    for (const Node* sp : points) {
      const int64_t v = atol(sp->value.c_str());
      if (v <= bounds.back() || v >= A)
        return L.refuse("slice_point " + std::to_string(v) + " is not increasing inside (0, " + std::to_string(A) + ")");
      bounds.push_back(v);
    }
  } else {
    if (A % ntop) return L.refuse(std::to_string(ntop) + " tops do not evenly divide slice axis " + std::to_string(A));
    for (int64_t t = 1; t < ntop; ++t) bounds.push_back(t * (A / ntop));
  }
  bounds.push_back(A);
  L.rec.axis = axis;
  for (int64_t t = 0; t < ntop; ++t) {
    Shape s = in;
    s[axis] = bounds[t + 1] - bounds[t];
    L.set_top(t, s);
    L.rec.slice_begin.push_back(bounds[t]);
    L.rec.slice_end.push_back(bounds[t + 1]);
  }
  return true;
}

bool contrastive_loss(Layer& L, std::vector<Shape>*) {  // contrastive_loss_layer.cpp LayerSetUp and LossLayer::Reshape
  Shape a, b, sim;
  if (L.rec.bottoms.size() != 3) return L.refuse("needs 3 bottoms (a, b, sim)");
  if (!L.bottom(0, &a) || !L.bottom(1, &b) || !L.bottom(2, &sim)) return false;
  auto legacy = [](const Shape& s, size_t i) { return i < s.size() ? s[i] : int64_t{1}; };  // Blob::LegacyShape
  if (a.empty() || a.size() > 4 || b.size() != a.size() || sim.empty() || sim.size() > 4)
    return L.refuse("bottoms must have 1 to 4 axes, a and b as many");
  if (b[0] != a[0] || sim[0] != a[0]) return L.refuse("a, b and sim must have the same first dimension");
  if (legacy(a, 1) != legacy(b, 1)) return L.refuse("a and b must have the same channels");
  if (legacy(a, 2) != 1 || legacy(a, 3) != 1 || legacy(b, 2) != 1 || legacy(b, 3) != 1)
    return L.refuse("a and b must be N x C (x 1 x 1)");
  if (legacy(sim, 1) != 1 || legacy(sim, 2) != 1 || legacy(sim, 3) != 1) return L.refuse("sim must hold one value per pair");
  if (const Node* p = L.node.first("contrastive_loss_param")) {
    L.rec.margin = static_cast<float>(p->num("margin", 1.0));
    L.rec.legacy_version = p->boolean("legacy_version", false);
  }
  L.set_tops(Shape{});
  return true;
}

bool loss(Layer& L, std::vector<Shape>*) {  // and Accuracy: scalar tops
  if (const Node* p = L.node.first("hinge_loss_param")) {  // caffe.proto HingeLossParameter.Norm: L1 = 1, L2 = 2
    L.rec.hinge_norm = p->str("norm", "L1");
    if (L.rec.hinge_norm == "1") L.rec.hinge_norm = "L1";
    if (L.rec.hinge_norm == "2") L.rec.hinge_norm = "L2";
  }
  L.set_tops(Shape{});
  return true;
}

bool softmax_loss(Layer& L, std::vector<Shape>* params) {  // softmax_loss_layer.cpp Reshape: the class axis
  Shape in;
  const Node* p = L.node.first("softmax_param");
  if (!L.rec.bottoms.empty() && L.blobs.count(L.rec.bottoms[0]) && L.bottom(0, &in) &&
      !canonical_axis(L, p ? p->integer("axis", 1) : 1, static_cast<int64_t>(in.size()), &L.rec.axis))
    return false;
  return loss(L, params);
}
bool silence(Layer&, std::vector<Shape>*) { return true; }

// The layer types the parser understands.  A new type needs a rule and a row here, and a row in native_producer.cpp's
// table if the built-in engine runs it.
const struct { const char* type; Rule rule; } kRules[] = {
    {"MemoryData", memory_data}, {"CoSData", cos_data}, {"Input", input},
    {"Convolution", convolution}, {"Deconvolution", convolution}, {"Pooling", pooling}, {"InnerProduct", inner_product},
    {"ReLU", same_shape}, {"LRN", same_shape}, {"Dropout", same_shape}, {"Sigmoid", same_shape}, {"TanH", same_shape},
    {"Softmax", same_shape}, {"Power", same_shape}, {"AbsVal", same_shape}, {"BNLL", same_shape}, {"ELU", same_shape},
    {"Exp", same_shape}, {"Log", same_shape}, {"Threshold", same_shape}, {"PReLU", prelu},
    {"Split", split}, {"Eltwise", eltwise}, {"Scale", scale}, {"Flatten", flatten}, {"Concat", concat},
    {"Embed", embed}, {"Reshape", reshape}, {"RNN", rnn}, {"MVN", mvn}, {"Crop", crop}, {"SPP", spp},
    {"Tile", tile},
    {"SoftmaxWithLoss", softmax_loss}, {"Accuracy", loss}, {"EuclideanLoss", loss}, {"SigmoidCrossEntropyLoss", loss},
    {"HingeLoss", loss}, {"MultinomialLogisticLoss", loss},
    {"BatchNorm", batch_norm}, {"Slice", slice}, {"ContrastiveLoss", contrastive_loss}, {"Silence", silence},
};

struct ParamOwners {
  std::map<std::string, int> by_name;  // ParamSpec.name -> the learnable blob that owns it
  std::vector<bool> has_lr, has_decay;  // per learnable blob: lr_mult / decay_mult set explicitly
};

// net.cpp AppendParam for the learnable blobs of one layer, of shapes `params`: an anonymous param, or the first use of
// a name, owns a learnable blob; a later use of the name shares the owner's.
bool append_params(const Node& layer, const std::vector<Shape>& params, ParamOwners* owners, SolverSpec* spec,
                   NetLayer* rec, std::string* err) {
  auto pspecs = layer.all("param");
  for (size_t i = 0; i < params.size(); ++i) {
    const Node* ps = i < pspecs.size() ? pspecs[i] : nullptr;
    const std::string pname = ps ? ps->str("name", "") : "";
    auto owner = pname.empty() ? owners->by_name.end() : owners->by_name.find(pname);
    if (owner == owners->by_name.end()) {
      if (!pname.empty()) owners->by_name[pname] = static_cast<int>(spec->counts.size());
      rec->blobs.push_back(static_cast<int>(spec->counts.size())), rec->shared.push_back(false);
      spec->counts.push_back(shape_count(params[i]));
      // ParamSpec defaults lr_mult = 1, decay_mult = 1 (caffe.proto:297-304)
      spec->lr_mult.push_back(ps ? static_cast<float>(ps->num("lr_mult", 1.0)) : 1.0f);
      spec->decay_mult.push_back(ps ? static_cast<float>(ps->num("decay_mult", 1.0)) : 1.0f);
      owners->has_lr.push_back(ps && ps->first("lr_mult")), owners->has_decay.push_back(ps && ps->first("decay_mult"));
      spec->blob_names.push_back(rec->name + "." + std::to_string(i));
      spec->layer_names.push_back(rec->name);
      spec->layer_types.push_back(rec->type);
      spec->shapes.push_back(params[i]);
      spec->param_index.push_back(static_cast<int>(i));
      continue;
    }
    const int k = owner->second;
    const std::string share = "Cannot share param '" + pname + "' owned by layer '" + spec->layer_names[k] +
                              "' with layer '" + rec->name + "'; ";
    const std::string mode = ps->str("share_mode", "STRICT");
    if (mode == "PERMISSIVE" || mode == "1") {
      if (spec->counts[k] != shape_count(params[i])) {
        *err = share + "count mismatch.  Owner layer param shape is " + shape_string(spec->shapes[k]) +
               "; sharing layer shape is " + shape_string(params[i]);
        return false;
      }
    } else if (spec->shapes[k] != params[i]) {
      *err = share + "shape mismatch.  Owner layer param shape is " + shape_string(spec->shapes[k]) +
             "; sharing layer expects shape " + shape_string(params[i]);
      return false;
    }
    // the first explicit lr_mult / decay_mult, by the owner or a sharer, is the blob's; a different later one is an error
    struct Mult { const char* field; std::vector<float>* value; std::vector<bool>* set; };
    for (const Mult& m : {Mult{"lr_mult", &spec->lr_mult, &owners->has_lr},
                          Mult{"decay_mult", &spec->decay_mult, &owners->has_decay}}) {
      if (!ps->first(m.field)) continue;
      const float v = static_cast<float>(ps->num(m.field, 1.0));
      if ((*m.set)[k] && v != (*m.value)[k]) {
        *err = "Shared param '" + pname + "' has mismatched " + m.field + ".";
        return false;
      }
      (*m.set)[k] = true;
      (*m.value)[k] = v;
    }
    rec->blobs.push_back(k);
    rec->shared.push_back(true);
    spec->shared.push_back(SharedParam{rec->name, rec->type, static_cast<int>(i), k, static_cast<int>(spec->counts.size())});
  }
  return true;
}

// `out` (optional) receives every TRAIN-phase layer with its blob shapes and the parameters the native producer reads.
// `net_file` is the prototxt the net was read from ("" for text).
bool net_layout(const Node& net, const std::string& net_file, SolverSpec* spec, std::vector<NetLayer>* out,
                std::string* err) {
  std::map<std::string, Shape> blobs;
  ParamOwners owners;
  bool first_data = true;
  auto record = [&](NetLayer& rec) {
    if (!out) return;
    for (const std::string& t : rec.tops) rec.top_shapes.push_back(blobs.count(t) ? blobs[t] : Shape());
    out->push_back(rec);
  };
  if (out) out->clear();
  spec->inputs.clear(), spec->counts.clear(), spec->lr_mult.clear(), spec->decay_mult.clear(), spec->shared.clear();
  spec->blob_names.clear(), spec->layer_names.clear(), spec->layer_types.clear(), spec->shapes.clear(), spec->param_index.clear();
  spec->net_name = net.str("name");
  {  // the legacy net-level "input:" blobs, each with an "input_shape" or four "input_dim"s, as one Input layer
    NetLayer rec;
    rec.name = "input", rec.type = "Input";
    Layer L{net, rec, blobs, err, spec, net_file, first_data};
    auto inputs = net.all("input"), shapes = net.all("input_shape"), dims = net.all("input_dim");
    for (size_t i = 0; i < inputs.size(); ++i) {
      Shape s;
      if (i < shapes.size()) for (const Node* d : shapes[i]->all("dim")) s.push_back(atol(d->value.c_str()));
      else for (size_t k = 4 * i; k < 4 * i + 4 && k < dims.size(); ++k) s.push_back(atol(dims[k]->value.c_str()));
      rec.tops.push_back(inputs[i]->value);
      data_top(L, i, s, nullptr);
    }
    if (!inputs.empty()) record(rec);
  }
  auto layers = net.all("layer");
  if (layers.empty() && !net.all("layers").empty()) {
    *err = "V1 'layers' net definitions are not supported";
    return false;
  }
  for (const Node* node : layers) {
    if (!in_train_phase(*node)) continue;
    NetLayer rec;
    rec.name = node->str("name"), rec.type = node->str("type");
    for (const Node* b : node->all("bottom")) rec.bottoms.push_back(b->value);
    for (const Node* t : node->all("top")) rec.tops.push_back(t->value);
    for (const std::string& b : rec.bottoms) rec.bottom_shapes.push_back(blobs.count(b) ? blobs[b] : Shape());
    rec.has_loss_param = node->first("loss_param") != nullptr;
    if (const Node* lw = node->first("loss_weight")) rec.loss_weight = static_cast<float>(atof(lw->value.c_str()));
    Rule rule = nullptr;
    for (const auto& row : kRules)
      if (rec.type == row.type) rule = row.rule;
    if (!rule) {
      *err = "layer '" + rec.name + "' of type '" + rec.type +
             "' is not understood by the layout parser; pass the layout with cos_net_allocate_desc";
      return false;
    }
    Layer L{*node, rec, blobs, err, spec, net_file, first_data};
    std::vector<Shape> params;
    if (!rule(L, &params) || !append_params(*node, params, &owners, spec, &rec, err)) return false;
    record(rec);
  }
  return true;
}

bool parse_solver(const std::string& solver_path, SolverSpec* spec, std::vector<NetLayer>* layers, std::string* err) {
  std::string text;
  if (!read_file(solver_path, &text)) {
    *err = "cannot read solver file '" + solver_path + "'";
    return false;
  }
  Node s;
  TextParser tp(text);
  if (!tp.parse(&s, err)) return false;
  spec->lr_policy = s.str("lr_policy", "fixed");
  spec->base_lr = static_cast<float>(s.num("base_lr", 0.0));
  spec->gamma = static_cast<float>(s.num("gamma", 0.0));
  spec->power = static_cast<float>(s.num("power", 0.0));
  spec->stepsize = static_cast<int>(s.integer("stepsize", 0));
  spec->stepvalues.clear();
  for (const Node* v : s.all("stepvalue")) spec->stepvalues.push_back(atoi(v->value.c_str()));
  spec->max_iter = static_cast<int>(s.integer("max_iter", 0));
  spec->momentum = static_cast<float>(s.num("momentum", 0.0));
  spec->weight_decay = static_cast<float>(s.num("weight_decay", 0.0));
  // repeated test_iter: the reference reads test_iter(0) (CaffeNet.cpp getTestIter)
  spec->test_iter = static_cast<int>(s.integer("test_iter", 0));
  spec->test_interval = static_cast<int>(s.integer("test_interval", 0));
  spec->snapshot_prefix = s.str("snapshot_prefix", "");
  spec->regularization_type = s.str("regularization_type", "L2");
  spec->iter_size = static_cast<int>(s.integer("iter_size", 1));
  spec->clip_gradients = static_cast<float>(s.num("clip_gradients", -1.0));
  spec->solver_mode_gpu = s.str("solver_mode", "GPU") != "CPU";
  spec->snapshot_hdf5 = s.str("snapshot_format", "BINARYPROTO") == "HDF5";
  spec->random_seed = s.integer("random_seed", -1);
  spec->solver_file = solver_path;
  spec->type = s.str("type", "");
  if (spec->type.empty()) spec->type = s.str("solver_type", "SGD");  // deprecated enum field
  if (spec->type != "SGD" && spec->type != "Adam" && spec->type != "ADAM") {
    *err = "solver type '" + spec->type + "' is not on the accelerated path (only SGD with momentum is)";
    return false;
  }
  if (spec->type == "ADAM") spec->type = "Adam";  // deprecated enum spelling (caffe.proto SolverType)
  spec->solver_type = spec->type == "Adam" ? 1 : 0;
  spec->momentum2 = static_cast<float>(s.num("momentum2", 0.999));
  spec->delta = static_cast<float>(s.num("delta", 1e-8));
  if (spec->regularization_type != "L2" && spec->regularization_type != "L1") {
    *err = "Unknown regularization type: " + spec->regularization_type;  // sgd_solver.cpp:169-171
    return false;
  }
  if (spec->iter_size < 1) {  // solver.cpp:37-38 CHECK_GE(iter_size, 1) (caffe.proto: iter_size default 1)
    *err = "iter_size must be >= 1 (got " + std::to_string(spec->iter_size) + ")";
    return false;
  }
  if (spec->clip_gradients >= 0.f) {
    *err = "clip_gradients is not supported";
    return false;
  }
  // locate the net definition
  if (const Node* inl = s.first("net_param") ? s.first("net_param") : s.first("train_net_param")) {
    return net_layout(*inl, solver_path, spec, layers, err) && check_solver_layout(*spec, err);
  }
  std::string net_path = s.str("net", "");
  if (net_path.empty()) net_path = s.str("train_net", "");
  if (net_path.empty()) {
    *err = "solver file names no net (net / train_net / net_param)";
    return false;
  }
  // as given, then relative to the solver file's directory, then by basename there
  const std::string net_file = find_relative_file(net_path, solver_path);
  std::string net_text;
  if (net_file.empty() || !read_file(net_file, &net_text)) {
    *err = "cannot read net file '" + net_path + "' named by '" + solver_path + "'";
    return false;
  }
  Node net;
  TextParser np(net_text);
  if (!np.parse(&net, err)) return false;
  return net_layout(net, net_file, spec, layers, err) && check_solver_layout(*spec, err);
}

}  // namespace

std::string find_relative_file(const std::string& path, const std::string& relative_to) {
  auto opens = [](const std::string& p) { return static_cast<bool>(std::ifstream(p.c_str(), std::ios::binary)); };
  if (opens(path)) return path;
  size_t slash = relative_to.find_last_of('/');
  std::string dir = slash == std::string::npos ? "." : relative_to.substr(0, slash);
  if (opens(dir + "/" + path)) return dir + "/" + path;
  size_t s2 = path.find_last_of('/');
  if (s2 != std::string::npos && opens(dir + "/" + path.substr(s2 + 1))) return dir + "/" + path.substr(s2 + 1);
  return "";
}

bool parse_train_net(const std::string& path, SolverSpec* spec, std::vector<NetLayer>* layers, std::string* err) {
  std::string text;
  if (!read_file(path, &text)) {
    *err = "cannot read prototxt '" + path + "'";
    return false;
  }
  Node top;
  TextParser tp(text);
  if (!tp.parse(&top, err)) return false;
  if (!top.all("layer").empty() || !top.all("layers").empty() || !top.all("input").empty())
    return net_layout(top, path, spec, layers, err);
  return parse_solver(path, spec, layers, err);
}

bool parse_solver_prototxt(const std::string& solver_path, SolverSpec* spec, std::string* err) {
  return parse_solver(solver_path, spec, nullptr, err);
}

bool check_solver_layout(const SolverSpec& spec, std::string* err) {
  uint64_t n = 0;
  for (int64_t c : spec.counts) n += static_cast<uint64_t>(c);
  if (spec.solver_type == 1 && n == 0) {
    *err = "solver type 'Adam' needs learnable parameters; for a net without any, only SGD is on the accelerated "
           "path (with no history blobs, its Adam and SGD solver states could not be told apart)";
    return false;
  }
  return true;
}

}  // namespace cosb
