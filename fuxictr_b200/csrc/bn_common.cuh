// bn_common.cuh — the batch-statistics finalize nn.BatchNorm1d does in training mode, shared by Dice (attention.cu)
// and FinalNet's factorized-interaction kernels (finalnet.cu).
//
// From the fp64 column sums s1 = sum_m x and s2 = sum_m x^2 over M rows: the mean and the rstd of the biased
// variance, and, when running_mean is not NULL, the running statistics updated with the unbiased variance,
//   running = (1 - momentum) running + momentum stat.
#pragma once
#include "b2_common.cuh"

__device__ __forceinline__ void b2_bn_finalize(double s1, double s2, int64_t M, float eps, float momentum,
                                               float* mean, float* rstd, float* running_mean, float* running_var) {
  const double mu = s1 / (double) M;
  double var = s2 / (double) M - mu * mu;
  if (var < 0.0) var = 0.0;
  *mean = (float) mu;
  *rstd = (float) (1.0 / sqrt(var + (double) eps));
  if (running_mean != nullptr) {
    const double unbiased = (M > 1) ? var * (double) M / (double) (M - 1) : var;
    *running_mean = (1.f - momentum) * *running_mean + momentum * (float) mu;
    *running_var = (1.f - momentum) * *running_var + momentum * (float) unbiased;
  }
}
