// data_transform.cu -- see data_transform.hpp.
#include "data_transform.hpp"

#include <stdio.h>

#include <sstream>

#include "caffe_proto_io.hpp"
#include "fused_sync_sgd.hpp"

namespace cosb {
namespace {

constexpr uint64_t kPhi = 0x9e3779b97f4a7c15ULL;
constexpr int kThreads = 128;     // one output row of one channel per pass (CaffeNet: 227 columns in two)
constexpr int kRowsPerBlock = 8;  // output rows per block: the draws and the launch are paid once for 8 rows

__host__ __device__ __forceinline__ uint32_t draw(uint64_t key, int n, int j, uint32_t range) {
  return static_cast<uint32_t>(mix64(key + (static_cast<uint64_t>(n) * 4 + static_cast<uint64_t>(j)) * kPhi) >> 32) %
         range;
}

struct TransformArgs {
  const void* in;
  float* out;
  const float* mean;  // C x H x W of the input, or null
  int C, H, W, Ho, Wo;
  int crop, mirror, nmean;
  float scale;
  uint64_t key;
  float mean_values[kMaxMeanValues];
};

// Stages src[0, L) in shared memory: the body between the first and last 4-byte boundary of src moves as words.
__device__ __forceinline__ void stage_row(const uint8_t* src, int L, uint8_t* dst) {
  const int head = static_cast<int>((4 - (reinterpret_cast<uintptr_t>(src) & 3)) & 3);
  const int lead = head < L ? head : L;
  const int nw = (L - lead) >> 2;
  const uint32_t* body = reinterpret_cast<const uint32_t*>(src + lead);
  for (int i = threadIdx.x; i < lead; i += blockDim.x) dst[i] = src[i];
  for (int i = threadIdx.x; i < nw; i += blockDim.x) {
    const uint32_t v = __ldg(body + i);
    uint8_t* d = dst + lead + 4 * i;
    d[0] = static_cast<uint8_t>(v), d[1] = static_cast<uint8_t>(v >> 8);
    d[2] = static_cast<uint8_t>(v >> 16), d[3] = static_cast<uint8_t>(v >> 24);
  }
  for (int i = lead + 4 * nw + threadIdx.x; i < L; i += blockDim.x) dst[i] = src[i];
}

// One block per kRowsPerBlock output rows of one image: Caffe's element loop for those rows, all channels.  The u8
// path copies each crop row (Wo x C interleaved bytes) to shared memory with aligned 4-byte loads; then the threads
// write consecutive output columns of one channel at a time, so both the reads and the fp32 stores are coalesced.
// Caffe's cv::Mat path draws per image (n); its Blob path draws once per batch (n = 0).
template <bool kU8>
__global__ void __launch_bounds__(kThreads) data_transform_kernel(const TransformArgs a) {
  extern __shared__ uint32_t row_words[];
  uint8_t* row = reinterpret_cast<uint8_t*>(row_words);
  const int row_blocks = (a.Ho + kRowsPerBlock - 1) / kRowsPerBlock;
  const int n = blockIdx.x / row_blocks, h0 = (blockIdx.x % row_blocks) * kRowsPerBlock;
  const int dn = kU8 ? n : 0;
  const bool mirror = a.mirror && draw(a.key, dn, 0, 2);
  const int h_off = a.crop ? static_cast<int>(draw(a.key, dn, 1, static_cast<uint32_t>(a.H - a.crop + 1))) : 0;
  const int w_off = a.crop ? static_cast<int>(draw(a.key, dn, 2, static_cast<uint32_t>(a.W - a.crop + 1))) : 0;
  const int h_end = h0 + kRowsPerBlock < a.Ho ? h0 + kRowsPerBlock : a.Ho;
  for (int h = h0; h < h_end; ++h) {
    const int hs = h_off + h;
    if (kU8) {
      if (h > h0) __syncthreads();  // every thread is done with the previous row
      stage_row(static_cast<const uint8_t*>(a.in) + ((static_cast<int64_t>(n) * a.H + hs) * a.W + w_off) * a.C,
                a.Wo * a.C, row);
      __syncthreads();
    }
    for (int c = 0; c < a.C; ++c) {
      const float mv = a.nmean ? a.mean_values[a.nmean == 1 ? 0 : c] : 0.f;
      for (int w = threadIdx.x; w < a.Wo; w += blockDim.x) {
        // mirrored: output column w holds input column Wo-1-w (Caffe writes width-1-w from w)
        const int ws = mirror ? a.Wo - 1 - w : w;
        const float x = kU8 ? static_cast<float>(row[ws * a.C + c])
                            : __ldg(static_cast<const float*>(a.in) +
                                    ((static_cast<int64_t>(n) * a.C + c) * a.H + hs) * a.W + w_off + ws);
        float v;
        if (a.mean) {
          v = __fmul_rn(__fsub_rn(x, __ldg(a.mean + (static_cast<int64_t>(c) * a.H + hs) * a.W + w_off + ws)),
                        a.scale);
        } else if (a.nmean) {
          v = __fmul_rn(__fsub_rn(x, mv), a.scale);
        } else {
          v = __fmul_rn(x, a.scale);
        }
        a.out[((static_cast<int64_t>(n) * a.C + c) * a.Ho + h) * a.Wo + w] = v;
      }
    }
  }
}

std::string shape_str(const std::vector<int64_t>& s) {
  std::ostringstream os;
  for (size_t i = 0; i < s.size(); ++i) os << (i ? "x" : "") << s[i];
  return s.empty() ? "scalar" : os.str();
}

std::string num_str(float v) {
  char b[32];
  snprintf(b, sizeof b, "%.9g", static_cast<double>(v));
  return b;
}

}  // namespace

uint64_t transform_key(int64_t seed, int rank, int input, int iter, int pass) {
  const uint64_t s = seed < 0 ? 0 : static_cast<uint64_t>(seed);
  uint64_t k = mix64(s * kPhi + static_cast<uint64_t>(static_cast<int64_t>(rank)));
  k = mix64(k + static_cast<uint64_t>(static_cast<int64_t>(input)));
  k = mix64(k + static_cast<uint64_t>(static_cast<int64_t>(iter)));
  return mix64(k + static_cast<uint64_t>(static_cast<int64_t>(pass)));
}

uint32_t transform_draw(uint64_t key, int n, int j, uint32_t range) { return draw(key, n, j, range); }

std::string check_transform_args(const void* in, int format, int num, int channels, int height, int width,
                                 const float* out, int crop_size, const float* mean, const float* mean_values,
                                 int nmean) {
  if (!in || !out) return "in and out must not be NULL";
  if (format != kRawF32Nchw && format != kRawU8Nhwc)
    return "format " + std::to_string(format) + " is neither COS_RAW_F32_NCHW nor COS_RAW_U8_NHWC";
  if (num < 1 || channels < 1 || height < 1 || width < 1) return "num, channels, height and width must be positive";
  if (crop_size < 0 || crop_size > height || crop_size > width)
    return "crop_size " + std::to_string(crop_size) + " must be in [0, min(height, width)]";
  if (mean && nmean) return "Cannot specify mean_file and mean_value at the same time";
  if (nmean < 0 || (nmean && !mean_values)) return "mean_values is NULL";
  if (nmean && nmean != 1 && nmean != channels)
    return "Specify either 1 mean_value or as many as channels: " + std::to_string(channels);
  if (nmean > kMaxMeanValues) return "at most " + std::to_string(kMaxMeanValues) + " mean values";
  const int64_t wo = crop_size ? crop_size : width;
  if (format == kRawU8Nhwc && wo * channels > kMaxTransformRowBytes)
    return "an 8-bit crop row of " + std::to_string(wo * channels) + " bytes exceeds " +
           std::to_string(kMaxTransformRowBytes);
  const int64_t ho = crop_size ? crop_size : height;
  if (static_cast<int64_t>(num) * ho > 0x7fffffff) return "num x output height exceeds the grid";
  return "";
}

cudaError_t launch_data_transform(const void* in, int format, int num, int channels, int height, int width, float* out,
                                  int crop_size, bool mirror, const float* mean, const float* mean_values, int nmean,
                                  float scale, uint64_t key, cudaStream_t stream) {
  TransformArgs a;
  a.in = in, a.out = out, a.mean = mean;
  a.C = channels, a.H = height, a.W = width;
  a.Ho = crop_size ? crop_size : height, a.Wo = crop_size ? crop_size : width;
  a.crop = crop_size, a.mirror = mirror ? 1 : 0, a.nmean = mean ? 0 : nmean;
  a.scale = scale, a.key = key;
  for (int i = 0; i < kMaxMeanValues; ++i) a.mean_values[i] = i < a.nmean ? mean_values[i] : 0.f;
  const int row_blocks = (a.Ho + kRowsPerBlock - 1) / kRowsPerBlock;
  const unsigned grid = static_cast<unsigned>(static_cast<int64_t>(num) * row_blocks);
  if (format == kRawU8Nhwc) {
    const size_t smem = (static_cast<size_t>(a.Wo) * channels + 3) & ~static_cast<size_t>(3);
    data_transform_kernel<true><<<grid, kThreads, smem, stream>>>(a);
  } else {
    data_transform_kernel<false><<<grid, kThreads, 0, stream>>>(a);
  }
  return cudaGetLastError();
}

bool resolve_input_transforms(const SolverSpec& spec, std::vector<InputTransform>* out, std::string* err) {
  out->clear();
  for (const StagedInput& in : spec.inputs) {
    InputTransform r;
    r.input = in;
    const TransformSpec& t = in.transform;
    auto refuse = [&](const std::string& why) {
      *err = "layer '" + in.layer + "' (" + in.type + "), top '" + in.top + "': " + why;
      return false;
    };
    if (t.present) {
      if (in.shape.size() != 4) return refuse("transform_param needs an N x C x H x W top, not " + shape_str(in.shape));
      const int64_t C = in.shape[1], H = in.shape[2], W = in.shape[3];
      if (!t.mean_file.empty() && !t.mean_values.empty())
        return refuse("Cannot specify mean_file and mean_value at the same time");
      if (!t.mean_values.empty() && t.mean_values.size() != 1 && static_cast<int64_t>(t.mean_values.size()) != C)
        return refuse("Specify either 1 mean_value or as many as channels: " + std::to_string(C));
      if (t.mean_values.size() > static_cast<size_t>(kMaxMeanValues))
        return refuse("at most " + std::to_string(kMaxMeanValues) + " mean values");
      if (t.crop_size < 0 || (t.crop_size && (t.crop_size != H || t.crop_size != W)))
        return refuse("crop_size " + std::to_string(t.crop_size) + " must equal the top's height and width (" +
                      std::to_string(H) + "x" + std::to_string(W) + ")");
      if (!t.mean_file.empty()) {
        r.mean_path = find_relative_file(t.mean_file, t.net_file);
        if (r.mean_path.empty()) return refuse("cannot open mean_file '" + t.mean_file + "'");
        ParsedBlob b;
        std::string why;
        if (!read_blobproto(r.mean_path, &b, &why)) return refuse("mean_file: " + why);
        if (b.shape.size() > 4)
          return refuse("mean_file '" + r.mean_path + "' has " + shape_str(b.shape) + ", more than 4 axes");
        auto legacy = [&](size_t i) { return i < b.shape.size() ? b.shape[i] : int64_t(1); };  // Blob::LegacyShape
        if (legacy(0) != 1)
          return refuse("mean_file '" + r.mean_path + "' has num " + std::to_string(legacy(0)) + "; it must be 1");
        if (legacy(1) != C)
          return refuse("mean_file '" + r.mean_path + "' has " + std::to_string(legacy(1)) + " channels, the top " +
                        std::to_string(C));
        r.mean_shape = {legacy(1), legacy(2), legacy(3)};
        r.mean = std::move(b.data);
      }
    }
    out->push_back(std::move(r));
  }
  return true;
}

std::string input_transform_plan_text(const std::vector<InputTransform>& inputs) {
  std::ostringstream os;
  for (size_t i = 0; i < inputs.size(); ++i) {
    const InputTransform& r = inputs[i];
    const TransformSpec& t = r.input.transform;
    os << "input " << i << " " << r.input.top << " layer=" << r.input.layer << " shape=" << shape_str(r.input.shape);
    if (!t.present) {
      os << " transform=none\n";
      continue;
    }
    os << " scale=" << num_str(t.scale) << " mirror=" << (t.mirror ? 1 : 0) << " crop=" << t.crop_size << " mean=";
    if (!r.mean_path.empty()) {
      os << "file:" << r.mean_path << "[" << shape_str(r.mean_shape) << "]";
    } else if (!t.mean_values.empty()) {
      os << "values:";
      for (size_t k = 0; k < t.mean_values.size(); ++k) os << (k ? "," : "") << num_str(t.mean_values[k]);
    } else {
      os << "none";
    }
    os << "\n";
  }
  return os.str();
}

}  // namespace cosb
