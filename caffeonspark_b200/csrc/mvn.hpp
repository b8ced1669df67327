// mvn.hpp -- Caffe's MVN layer (mvn_layer.cu) for the gradient producer (mvn.cu, DESIGN.md section 14).
//
// x, y, dy, dx are `rows` contiguous rows of `dim` fp32 elements on the device (rows * dim < 2^31); each row is
// normalised on its own.
// With alpha = (float)(1.0 / dim) and every operation rounded once, as Forward_gpu and Backward_gpu round them:
//   forward   mu = Sx * alpha, y = x - mu; with normalize_variance var = Syy * alpha, s = powf(var, 0.5) + eps and
//             y = (x - mu) / s, where Sx = sum x and Syy = sum (x - mu)^2
//   backward  with normalize_variance dx = (dy + c * (y * A + B)) / s, c = (float)(-1.0 / dim), A = sum y * dy and
//             B = sum dy; mean-only dx = dy - B * alpha
// Only the order of the five row sums is the kernels' own: it is fixed by (rows, dim) alone, so results are bitwise
// identical from run to run, and no float atomics are used.  stats holds 5 * rows floats, each a row vector:
//   [0, rows) Sx, [rows, 2 rows) Syy, [2 rows, 3 rows) s   written by the forward (Syy = 0 and s = 1 mean-only)
//   [3 rows, 4 rows) A, [4 rows, 5 rows) B                  written by the backward (A = 0 mean-only)
// The backward reads s.  workspace is mvn_workspace_floats(rows, dim) floats (the long rows' chunk partials).
// The launchers only enqueue on `stream` (no allocation, synchronisation or device query).
//
// How a row maps onto the GPU depends on dim (and rows), with these thresholds:
//   dim <= kMvnLanesMaxDim                            next_pow2(dim) lanes of a warp per row (several rows per warp)
//   dim <= kMvnWarpMaxDim                             one warp per row
//   dim >= kMvnSplitMinDim and rows < kMvnSplitMaxRows the row is split into fixed chunks, one 256-thread block each;
//                                                     the chunk partials are added in chunk order
//   otherwise                                         one 256-thread block per row
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace cosb {

constexpr int64_t kMvnLanesMaxDim = 16, kMvnWarpMaxDim = 512, kMvnSplitMinDim = 16384, kMvnSplitMaxRows = 1024;
// the chunk of a split row: kMvnChunk elements, or more when the row would have more than kMvnMaxChunks chunks
constexpr int64_t kMvnChunk = 8192, kMvnMaxChunks = 1024;

enum class MvnRegime { kLanes, kWarp, kBlock, kSplit };
MvnRegime mvn_regime(int64_t rows, int64_t dim);
// the split regime's chunk length and count (chunk = dim, chunks = 1 in the others)
void mvn_chunks(int64_t rows, int64_t dim, int64_t* chunk, int64_t* chunks);
size_t mvn_workspace_floats(int64_t rows, int64_t dim);

cudaError_t mvn_forward(const float* x, float* y, float* stats, float* workspace, int64_t rows, int64_t dim,
                        bool normalize_variance, float eps, cudaStream_t stream);
cudaError_t mvn_backward(const float* y, const float* dy, float* dx, float* stats, float* workspace, int64_t rows,
                         int64_t dim, bool normalize_variance, cudaStream_t stream);

}  // namespace cosb
