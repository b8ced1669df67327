/*
 * adam_oracle.c -- CPU ORACLE for Adam solvers (test infrastructure, NOT product code).
 *
 * The Adam counterpart of sync_oracle.c's apply_update / step: AdamSolver::ComputeUpdateValue's CPU branch
 * (adam_solver.cpp) after the same on_start, scale, reduce-scatter and Regularize.  Linked together with
 * sync_oracle.c (oracle/adam.py builds both into oracle/_build/libadam_oracle.so) and compiled with the same
 * -ffp-contract=off -fno-fast-math, so every fp32 operation is rounded once.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "sync_oracle.h"
#include "../caffeonspark_b200/csrc/powf_half.h" /* only for cos_oracle_powf_half_check */

/* adam_solver.cpp:39-41: const int t = iter_ + 1; correction = std::sqrt(Dtype(1) - pow(beta2, t)) /
 * (Dtype(1.) - pow(beta1, t)).  pow(float, int) is the double overload, so everything right of the '=' is
 * double, rounded once to float by the assignment to const Dtype. */
float cos_oracle_adam_correction(float beta1, float beta2, int it) {
  const int t = it + 1;
  return (float)(sqrt((double)1.0f - pow((double)beta2, (double)t)) / ((double)1.0f - pow((double)beta1, (double)t)));
}

/* SGDSolver::ApplyUpdate (sgd_solver.cpp:102-116) with AdamSolver::ComputeUpdateValue, CPU branch
 * (adam_solver.cpp:26-75), per learnable blob k; Regularize exactly as in cos_oracle_apply_update_ex:
 *   local_rate = rate * lr_mult_k                                          :29
 *   caffe_cpu_axpby(N, 1-beta1, g, beta1, m)  = sscal + saxpy              :48-50   m = (1-b1)*g + (b1*m)
 *   caffe_mul(g, g -> t)                                                   :53-56   t = g*g
 *   caffe_cpu_axpby(N, 1-beta2, t, beta2, v)                               :57-59   v = (1-b2)*t + (b2*v)
 *   caffe_powx(v, 0.5 -> t)  = vsPowx = powf (mkl_alternate.hpp)           :62-64   t = powf(v, 0.5f)
 *   caffe_add_scalar(eps_hat, t)                                           :65      t = t + delta
 *   caffe_div(m, t -> t)                                                   :66-69   t = m / t
 *   caffe_cpu_scale(local_rate*correction, t -> g) = copy + sscal          :71-73   g = (lr*corr)*t
 *   Blob::Update: caffe_axpy(-1, g, w)                                              w = (-1*g) + w
 * history_[k] is m, history_[k + nblobs] is v (:34-36): here hist[i] and hist[P + i]. */
void cos_oracle_apply_update_adam(uint64_t begin, uint64_t end, uint64_t P, float* data, float* diff, float* hist,
                                  int nblobs, const int64_t* counts, const float* lr_mult, const float* decay_mult,
                                  float rate, float beta1, float beta2, float delta, float weight_decay, int l1,
                                  int it) {
  const float correction = cos_oracle_adam_correction(beta1, beta2, it);
  const float om1 = 1.0f - beta1, om2 = 1.0f - beta2;
  uint64_t blob_begin = 0;
  for (int k = 0; k < nblobs; ++k) {
    uint64_t blob_end = blob_begin + (uint64_t)counts[k];
    uint64_t lo = blob_begin > begin ? blob_begin : begin;
    uint64_t hi = blob_end < end ? blob_end : end;
    const float local_decay = weight_decay * decay_mult[k];
    const float local_rate = rate * lr_mult[k];
    const float lrc = local_rate * correction;
    for (uint64_t i = lo; i < hi; ++i) {
      float g = diff[i];
      float w = data[i];
      float m = hist[i];
      float v = hist[P + i];
      if (local_decay != 0.f) {
        float x = l1 ? (float)((0.f < w) - (w < 0.f)) : w;
        float t = local_decay * x;
        g = t + g;
      }
      m = beta1 * m;
      {
        float t = om1 * g;
        m = t + m;
      }
      float t = g * g;
      v = beta2 * v;
      {
        float u = om2 * t;
        v = u + v;
      }
      t = powf(v, 0.5f);
      t = t + delta;
      t = m / t;
      g = lrc * t;
      {
        float u = -1.0f * g;
        w = u + w;
      }
      diff[i] = g;
      hist[i] = m;
      hist[P + i] = v;
      data[i] = w;
    }
    blob_begin = blob_end;
  }
}

/* cos_oracle_step_ex with the Adam update (same on_start, scale and reduce-scatter). */
void cos_oracle_step_adam(int N, uint64_t P, float* const* data, float* const* diff, float* const* hist, int nblobs,
                          const int64_t* counts, const float* lr_mult, const float* decay_mult, float rate,
                          float beta1, float beta2, float delta, float weight_decay, int l1, int it) {
  if (N > 1) cos_oracle_all_gather(N, P, data);
  if (N > 1) {
    for (int r = 0; r < N; ++r) cos_oracle_scale(N, P, diff[r]);
    cos_oracle_reduce_scatter(N, P, diff);
  }
  for (int r = 0; r < N; ++r) {
    cos_oracle_apply_update_adam(0, P, P, data[r], diff[r], hist[r], nblobs, counts, lr_mult, decay_mult, rate,
                                 beta1, beta2, delta, weight_decay, l1, it);
  }
}

/* Over the bit patterns [lo, hi): counts[0] = inputs where powf(x, 0.5f) != sqrtf(x), counts[1] = inputs where
 * powf(x, 0.5f) differs from the update kernels' restatement (caffeonspark_b200/csrc/powf_half.h).  NaN results
 * compare equal to each other. */
void cos_oracle_powf_half_check(uint32_t lo, uint32_t hi, uint64_t* counts) {
  uint64_t vs_sqrt = 0, vs_device = 0;
  for (uint64_t u = lo; u < hi; ++u) {
    float x;
    uint32_t b = (uint32_t)u;
    memcpy(&x, &b, 4);
    const float a = powf(x, 0.5f), s = sqrtf(x), d = cos_powf_half(x);
    uint32_t ab, sb, db;
    memcpy(&ab, &a, 4);
    memcpy(&sb, &s, 4);
    memcpy(&db, &d, 4);
    if (ab != sb && !(isnan(a) && isnan(s))) ++vs_sqrt;
    if (ab != db && !(isnan(a) && isnan(d))) ++vs_device;
  }
  counts[0] = vs_sqrt;
  counts[1] = vs_device;
}

/* out[u - lo] = powf(x, 0.5f) for the bit patterns u in [lo, hi): the libm values the BatchNorm kernels' device
 * copy of powf_half.h is checked against.  Independent ranges may be filled from separate threads. */
void cos_oracle_powf_half_fill(uint32_t lo, uint32_t hi, float* out) {
  for (uint64_t u = lo; u < hi; ++u) {
    float x;
    uint32_t b = (uint32_t)u;
    memcpy(&x, &b, 4);
    out[u - lo] = powf(x, 0.5f);
  }
}
