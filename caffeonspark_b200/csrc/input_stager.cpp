// input_stager.cpp -- see input_stager.hpp.
#include "input_stager.hpp"

#include <sstream>

namespace cosb {
namespace {

std::string rt_err(const char* what, cudaError_t e) {
  std::ostringstream os;
  os << what << " failed: " << cudaGetErrorString(e);
  cudaGetLastError();
  return os.str();
}

#define COS_RT(call)                      \
  do {                                    \
    cudaError_t e__ = (call);             \
    if (e__ != cudaSuccess) {             \
      *err = rt_err(#call, e__);          \
      return false;                       \
    }                                     \
  } while (0)

std::string hw(int64_t h, int64_t w) { return std::to_string(h) + "x" + std::to_string(w); }

// Transform()'s size checks on one h x w image (data_transformer.cpp): a blob's (`noun` "raw"), or one ragged image's
// after its resize ("image", `which` naming it).  "" when it passes.
std::string check_size(int64_t h, int64_t w, const std::string& which, const char* noun, const InputTransform& t) {
  const std::vector<int64_t>& top = t.input.shape;
  const int64_t crop = t.input.transform.crop_size;
  if (crop) {
    if (h < crop || w < crop)
      return which + "Check failed: img_height >= crop_size (" + hw(h, w) + " vs. " + std::to_string(crop) + ")";
  } else if (h != top[2] || w != top[3]) {
    return which + "Check failed: img_height == height (" + noun + " " + hw(h, w) + ", top " + hw(top[2], top[3]) + ")";
  }
  if (!t.mean.empty() && (h != t.mean_shape[1] || w != t.mean_shape[2]))
    return which + "Check failed: img_height == data_mean_.height() (" + noun + " " + hw(h, w) + ", mean " +
           hw(t.mean_shape[1], t.mean_shape[2]) + ")";
  return "";
}

// DataTransformer's checks (Transform(cv::Mat) and Transform(Blob*)) on train_raw's input i.  "" when it passes.
std::string check_raw_input(const cos_raw_blob& b, const InputTransform& t, int i) {
  if (!b.data) return "data[" + std::to_string(i) + "] is NULL";
  if (b.format != kRawF32Nchw && b.format != kRawU8Nhwc && b.format != kRawU8Images)
    return "format " + std::to_string(b.format) + " is not COS_RAW_F32_NCHW, COS_RAW_U8_NHWC or COS_RAW_U8_IMAGES";
  const bool images = b.format == kRawU8Images;
  if (!images && (b.num < 1 || b.channels < 1 || b.height < 1 || b.width < 1))
    return "num, channels, height and width must be positive";
  const std::vector<int64_t>& top = t.input.shape;
  if (!t.active()) {
    int64_t want = 1;
    for (int64_t d : top) want *= d;
    if (images || b.format != kRawF32Nchw || static_cast<int64_t>(b.num) * b.channels * b.height * b.width != want)
      return "an input without transform_param must be COS_RAW_F32_NCHW with the top's " + std::to_string(want) +
             " elements";
    return "";
  }
  const int64_t crop = t.input.transform.crop_size;
  if (b.num != top[0]) return "raw num " + std::to_string(b.num) + " != the top's " + std::to_string(top[0]);
  if (b.channels != top[1])
    return "Check failed: channels == img_channels (" + std::to_string(top[1]) + " vs. " + std::to_string(b.channels) +
           ")";
  if (!images) {
    const std::string why = check_size(b.height, b.width, "", "raw", t);
    const int64_t row = (crop ? crop : b.width) * b.channels;
    if (why.empty() && b.format == kRawU8Nhwc && row > kMaxTransformRowBytes)
      return "an 8-bit crop row of " + std::to_string(row) + " bytes exceeds " + std::to_string(kMaxTransformRowBytes);
    return why;
  }
  // COS_RAW_U8_IMAGES: the caller's array of num images is read only now that num is the top's batch
  if (b.height < 0 || b.width < 0 || (b.height == 0) != (b.width == 0))
    return "resize target " + hw(b.height, b.width) + ": give both sides, or 0x0 for no resize";
  const int64_t wo = crop ? crop : top[3];
  if (wo > kMaxImageOutWidth)
    return "an output width of " + std::to_string(wo) + " exceeds " + std::to_string(kMaxImageOutWidth);
  const cos_raw_image* img = static_cast<const cos_raw_image*>(b.data);
  int64_t total = 0;
  for (int k = 0; k < b.num; ++k) {
    const std::string which = "image " + std::to_string(k) + ": ";
    if (!img[k].data) return which + "data is NULL";
    const int h = img[k].height, w = img[k].width;
    if (h < 1 || w < 1) return which + "height and width must be positive (" + hw(h, w) + ")";
    const std::string why = check_size(b.height ? b.height : h, b.height ? b.width : w, which, "image", t);
    if (!why.empty()) return why;
    int64_t bytes = 0;
    if (__builtin_mul_overflow(static_cast<int64_t>(h) * w, static_cast<int64_t>(b.channels), &bytes) ||
        __builtin_add_overflow(total, bytes, &total))
      return "the images' total byte count overflows";
  }
  return "";
}

}  // namespace

bool InputStager::create(int device, cudaStream_t compute, std::string* err) {
  device_ = device;
  compute_ = compute;
  COS_RT(cudaStreamCreateWithFlags(&copy_, cudaStreamNonBlocking));
  for (Stage& s : stages_) {
    COS_RT(cudaEventCreateWithFlags(&s.copied, cudaEventDisableTiming));
    COS_RT(cudaEventCreateWithFlags(&s.consumed, cudaEventDisableTiming));
  }
  return true;
}

void InputStager::release() {
  for (Stage& s : stages_) {
    s.inputs.clear();
    if (s.copied) cudaEventDestroy(s.copied);
    if (s.consumed) cudaEventDestroy(s.consumed);
    s.copied = s.consumed = nullptr;
  }
  means_.clear();
  if (copy_) cudaStreamDestroy(copy_);
  copy_ = nullptr;
}

bool InputStager::check_raw(const SolverSpec& spec, const cos_raw_blob* data, int ndata, std::string* err) {
  const bool first = raw_shapes_.empty();
  std::vector<InputTransform> resolved;
  if (first && !resolve_input_transforms(spec, &resolved, err)) return false;
  const std::vector<InputTransform>& tr = first ? resolved : transforms_;
  if (ndata != static_cast<int>(tr.size())) {
    *err = "train_raw: " + std::to_string(ndata) + " blobs for the net's " + std::to_string(tr.size()) +
           " staged inputs";
    return false;
  }
  for (int i = 0; i < ndata; ++i) {
    const cos_raw_blob& b = data[i];
    std::string why = check_raw_input(b, tr[i], i);
    const cos_raw_blob* s = first ? nullptr : &raw_shapes_[i];
    if (why.empty() && s &&
        (b.format != s->format || b.num != s->num || b.channels != s->channels || b.height != s->height ||
         b.width != s->width))
      why = "raw shape " + std::to_string(b.num) + "x" + std::to_string(b.channels) + "x" + hw(b.height, b.width) +
            " (format " + std::to_string(b.format) + ") differs from the first call's " + std::to_string(s->num) +
            "x" + std::to_string(s->channels) + "x" + hw(s->height, s->width) + " (format " +
            std::to_string(s->format) + ")";
    if (!why.empty()) {
      const StagedInput& in = tr[i].input;
      *err = "train_raw: layer '" + in.layer + "' (" + in.type + "), top '" + in.top + "': " + why;
      return false;
    }
  }
  if (!first) return true;
  // the means go to this net's device once; the first call's shapes are kept
  COS_RT(cudaSetDevice(device_));
  std::vector<DeviceBuffer> means(resolved.size());
  for (size_t i = 0; i < resolved.size(); ++i) {
    const size_t n = resolved[i].mean.size() * sizeof(float);
    cudaError_t e = means[i].grow(n, compute_);
    if (e == cudaSuccess && n) e = cudaMemcpy(means[i].get(), resolved[i].mean.data(), n, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      *err = rt_err("train_raw: mean upload", e);
      return false;
    }
  }
  transforms_ = std::move(resolved);
  means_ = std::move(means);
  raw_shapes_.assign(data, data + ndata);
  for (cos_raw_blob& s : raw_shapes_) s.data = nullptr;
  return true;
}

bool InputStager::stage(const cos_blob* data, const cos_raw_blob* raw, int nblobs, std::vector<cos_blob>* in,
                        std::string* err) {
  for (int i = 0; i < nblobs; ++i) {
    if (!(raw ? raw[i].data : data[i].data)) {
      *err = "data[" + std::to_string(i) + "] is NULL";
      return false;
    }
  }
  Stage& st = stages_[idx_];
  if (static_cast<int>(st.inputs.size()) < nblobs) st.inputs.resize(nblobs);
  // This stage was last read by step t-2: its H2D may only start once that step is done (device-side wait).
  if (st.consumed_valid) COS_RT(cudaStreamWaitEvent(copy_, st.consumed, 0));
  struct Piece {
    const void* host;
    size_t offset, bytes;
  };
  std::vector<Piece> pieces;
  *in = std::vector<cos_blob>(nblobs);
  for (int i = 0; i < nblobs; ++i) {
    Input& s = st.inputs[i];
    const cos_raw_blob* r = raw ? raw + i : nullptr;
    cos_blob b = r ? cos_blob{nullptr, r->num, r->channels, r->height, r->width} : data[i];
    // The host bytes: one piece, or one per image of a ragged batch, whose geometry table (offset, height, width per
    // image) is written to pinned memory once step t-2's copy of it has finished.
    const bool images = r && r->format == kRawU8Images;
    const size_t table = images ? static_cast<size_t>(b.num) * sizeof(ImageGeometry) : 0;
    size_t bytes = 0;
    pieces.clear();
    if (images) {
      COS_RT(s.geom_host.grow(table, compute_));
      COS_RT(cudaEventSynchronize(st.copied));
      const cos_raw_image* img = static_cast<const cos_raw_image*>(r->data);
      ImageGeometry* geom = static_cast<ImageGeometry*>(s.geom_host.get());
      for (int k = 0; k < b.num; ++k) {
        const size_t n = static_cast<size_t>(img[k].height) * img[k].width * b.channels;
        geom[k] = ImageGeometry{static_cast<int64_t>(bytes), img[k].height, img[k].width};
        pieces.push_back(Piece{img[k].data, bytes, n});
        bytes += n;
      }
    } else {
      bytes = static_cast<size_t>(b.num) * b.channels * b.height * b.width *
              (r && r->format == kRawU8Nhwc ? 1 : sizeof(float));
      pieces.push_back(Piece{r ? r->data : data[i].data, 0, bytes});
    }
    // An input with a transform_param lands in the raw set, and each pass transforms it into the fp32 set, which has
    // the top's height and width; every other input goes straight to the fp32 set.
    const bool transformed = r && transforms_[i].active();
    if (transformed) {
      const std::vector<int64_t>& top = transforms_[i].input.shape;
      b.height = static_cast<int>(top[2]), b.width = static_cast<int>(top[3]);
    }
    COS_RT(s.fp32.grow(static_cast<size_t>(b.num) * b.channels * b.height * b.width * sizeof(float), compute_));
    COS_RT(s.raw.grow(transformed ? bytes : 0, compute_));
    COS_RT(s.geom.grow(table, compute_));
    char* dst = static_cast<char*>(transformed ? s.raw.get() : s.fp32.get());
    for (const Piece& p : pieces)
      COS_RT(cudaMemcpyAsync(dst + p.offset, p.host, p.bytes, cudaMemcpyHostToDevice, copy_));
    if (images) COS_RT(cudaMemcpyAsync(s.geom.get(), s.geom_host.get(), table, cudaMemcpyHostToDevice, copy_));
    b.data = static_cast<const float*>(s.fp32.get());
    (*in)[i] = b;
  }
  COS_RT(cudaEventRecord(st.copied, copy_));
  COS_RT(cudaStreamWaitEvent(compute_, st.copied, 0));
  return true;
}

bool InputStager::transform(int64_t seed, int rank, int iter, int pass, std::string* err) {
  Stage& st = stages_[idx_];
  for (size_t i = 0; i < transforms_.size(); ++i) {
    const InputTransform& t = transforms_[i];
    if (!t.active()) continue;
    const TransformSpec& ts = t.input.transform;
    const cos_raw_blob& b = raw_shapes_[i];  // every call has the first call's shapes
    const Input& s = st.inputs[i];
    const float* mean = static_cast<const float*>(means_[i].get());
    const uint64_t key = transform_key(seed, rank, static_cast<int>(i), iter, pass);
    if (b.format == kRawU8Images) {
      const std::vector<int64_t>& top = t.input.shape;
      const bool file = mean != nullptr;
      COS_RT(launch_image_transform(static_cast<const uint8_t*>(s.raw.get()),
                                    static_cast<const ImageGeometry*>(s.geom.get()), b.num, b.channels, b.height,
                                    b.width, static_cast<float*>(s.fp32.get()), static_cast<int>(top[2]),
                                    static_cast<int>(top[3]), static_cast<int>(ts.crop_size), ts.mirror, mean,
                                    file ? static_cast<int>(t.mean_shape[1]) : 0,
                                    file ? static_cast<int>(t.mean_shape[2]) : 0, ts.mean_values.data(),
                                    static_cast<int>(ts.mean_values.size()), ts.scale, key, compute_));
      continue;
    }
    COS_RT(launch_data_transform(s.raw.get(), b.format, b.num, b.channels, b.height, b.width,
                                 static_cast<float*>(s.fp32.get()), static_cast<int>(ts.crop_size), ts.mirror, mean,
                                 ts.mean_values.data(), static_cast<int>(ts.mean_values.size()), ts.scale, key,
                                 compute_));
  }
  return true;
}

bool InputStager::mark_consumed(std::string* err) {
  Stage& st = stages_[idx_];
  COS_RT(cudaEventRecord(st.consumed, compute_));
  st.consumed_valid = true;
  idx_ ^= 1;
  return true;
}

bool InputStager::wait_copied(std::string* err) {
  COS_RT(cudaEventSynchronize(stages_[idx_ ^ 1].copied));
  return true;
}

}  // namespace cosb
