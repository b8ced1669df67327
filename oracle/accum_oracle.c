/*
 * accum_oracle.c -- CPU ORACLE for iter_size > 1 (gradient accumulation); test infrastructure, NOT product code.
 *
 * Solver::Step (solver.cpp:201-257) runs iter_size forward/backward passes whose gradients add up in diff_
 * (solver.cpp:221-224), then on_gradients_ready (scale + reduce-scatter) and ApplyUpdate, whose first call per blob
 * is SGDSolver::Normalize (sgd_solver.cpp:118-142):
 *   if (this->param_.iter_size() == 1) { return; }
 *   const Dtype accum_normalization = Dtype(1.) / this->param_.iter_size();
 *   caffe_scal(net_params[param_id]->count(), accum_normalization, diff);
 * Regularize and ComputeUpdateValue follow, for SGD and for Adam (AdamSolver inherits ApplyUpdate).  Linked with
 * sync_oracle.c and adam_oracle.c (oracle/accum.py builds oracle/_build/libaccum_oracle.so) with the same
 * -ffp-contract=off -fno-fast-math, so every fp32 operation is rounded once.
 */
#include <stdint.h>

#include "sync_oracle.h"

void cos_oracle_apply_update_adam(uint64_t begin, uint64_t end, uint64_t P, float* data, float* diff, float* hist,
                                  int nblobs, const int64_t* counts, const float* lr_mult, const float* decay_mult,
                                  float rate, float beta1, float beta2, float delta, float weight_decay, int l1,
                                  int it);

/* Dtype(1.) / iter_size: a float divided by an int, i.e. by (float)iter_size. */
float cos_oracle_accum_norm(int iter_size) { return 1.0f / (float)iter_size; }

/* One pass's Backward adding its gradient into diff_ (the layers accumulate: diff = g + diff). */
void cos_oracle_accumulate(uint64_t P, float* diff, const float* g) {
  for (uint64_t i = 0; i < P; ++i) diff[i] = g[i] + diff[i];
}

/* sgd_solver.cpp:118-142 Normalize: caffe_scal = cblas_sscal, diff[i] = accum_norm * diff[i], one rounding. */
void cos_oracle_normalize(uint64_t P, float* diff, float accum_norm) {
  for (uint64_t i = 0; i < P; ++i) diff[i] = accum_norm * diff[i];
}

/* The solver.cpp:221-224 loss: Dtype loss = 0; loss += ForwardBackward() per pass; loss /= iter_size. */
float cos_oracle_loss_mean(int passes, const float* losses) {
  float loss = 0.f;
  for (int i = 0; i < passes; ++i) loss += losses[i];
  loss /= (float)passes;
  return loss;
}

/* One Solver::Step after the passes: diff[r] holds rank r's accumulated gradient.  on_start (all-gather), scale,
 * reduce-scatter as cos_oracle_step_ex; then per rank Normalize (skipped for accum_norm == 1, i.e. iter_size 1)
 * and the SGD (adam == 0) or Adam (adam == 1; momentum is beta1, `it` the iteration before the step) update. */
void cos_oracle_step_accum(int N, uint64_t P, float* const* data, float* const* diff, float* const* hist, int nblobs,
                           const int64_t* counts, const float* lr_mult, const float* decay_mult, float rate,
                           float momentum, float weight_decay, int l1, float accum_norm, int adam, float beta2,
                           float delta, int it) {
  if (N > 1) cos_oracle_all_gather(N, P, data);
  if (N > 1) {
    for (int r = 0; r < N; ++r) cos_oracle_scale(N, P, diff[r]);
    cos_oracle_reduce_scatter(N, P, diff);
  }
  for (int r = 0; r < N; ++r) {
    if (accum_norm != 1.0f) cos_oracle_normalize(P, diff[r], accum_norm);
    if (adam) {
      cos_oracle_apply_update_adam(0, P, P, data[r], diff[r], hist[r], nblobs, counts, lr_mult, decay_mult, rate,
                                   momentum, beta2, delta, weight_decay, l1, it);
    } else {
      cos_oracle_apply_update_ex(0, P, data[r], diff[r], hist[r], nblobs, counts, lr_mult, decay_mult, rate, momentum,
                                 weight_decay, l1);
    }
  }
}
