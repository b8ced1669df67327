// data_transform.hpp -- Caffe's TRAIN-phase DataTransformer (data_transformer.cpp) on the device.
//
// The reference transforms every image on the CPU, in the JVM's transformer threads, before train() copies fp32 to
// the GPU (CaffeProcessor.scala:255-372).  Here the untransformed batch (8-bit NHWC images, or an fp32 NCHW blob) is
// staged and one sm_90a kernel applies crop, mirror, mean and scale with Caffe's arithmetic.  The random draws are
// a counter-based hash instead of Caffe's boost RNG (DESIGN.md, "Input transform on the device").
#ifndef COS_DATA_TRANSFORM_HPP_
#define COS_DATA_TRANSFORM_HPP_

#include <cuda_runtime_api.h>

#include <cstdint>
#include <string>
#include <vector>

#include "solver_spec.hpp"

namespace cosb {

constexpr int kRawF32Nchw = 0;  // COS_RAW_F32_NCHW
constexpr int kRawU8Nhwc = 1;   // COS_RAW_U8_NHWC
constexpr int kMaxMeanValues = 64;
constexpr int kMaxTransformRowBytes = 48 * 1024;  // one staged u8 crop row (crop x channels bytes)

// mix64(mix64(mix64(mix64(seed * phi + rank) + input) + iter) + pass); a negative seed counts as 0
uint64_t transform_key(int64_t seed, int rank, int input, int iter, int pass);
// one draw: uint32(mix64(key + (n * 4 + j) * phi) >> 32) % range (host copy of the kernel's)
uint32_t transform_draw(uint64_t key, int n, int j, uint32_t range);

// cos_data_transform's argument checks: "" when the call is valid
std::string check_transform_args(const void* in, int format, int num, int channels, int height, int width,
                                 const float* out, int crop_size, const float* mean, const float* mean_values,
                                 int nmean);
// Enqueues the transform (arguments already checked); mean_values is host memory.
cudaError_t launch_data_transform(const void* in, int format, int num, int channels, int height, int width, float* out,
                                  int crop_size, bool mirror, const float* mean, const float* mean_values, int nmean,
                                  float scale, uint64_t key, cudaStream_t stream);

// A staged input's transform_param, checked against its top, with its mean file read.
struct InputTransform {
  StagedInput input;
  std::string mean_path;             // the file read ("" without a mean file)
  std::vector<int64_t> mean_shape;   // channels, height, width of the mean blob
  std::vector<float> mean;           // host copy
  bool active() const { return input.transform.present; }
};
// Everything cos_input_transform_plan refuses, with the layer named.
bool resolve_input_transforms(const SolverSpec& spec, std::vector<InputTransform>* out, std::string* err);
std::string input_transform_plan_text(const std::vector<InputTransform>& inputs);

}  // namespace cosb
#endif
