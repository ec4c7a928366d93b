// The batch-statistics scheme shared by the training kernels (mdtc_train.cu, tcn_train.cu).  A launch runs
// TRAIN_SLICES CTAs for its row-sliced work, CTA z owning the fixed row slice z of the M = B * T rows.  A batch
// statistic (Sigma x, Sigma x^2 of the forward; Sigma g, Sigma g x_hat of the backward) is formed per slice in double,
// and every CTA of the next launch adds the slices in slice order in its prologue.  No atomics: equal inputs give
// equal bits.
#pragma once
#include <cuda_runtime.h>

namespace wekws {
namespace train {

constexpr int TRAIN_SLICES = 128;
constexpr int TRAIN_NT = 256;          // threads of every row-sliced CTA

struct Rows {
  long long r0, r1;
};
__device__ inline Rows slice_rows(long long M) {
  const long long rs = (M + TRAIN_SLICES - 1) / TRAIN_SLICES;
  const long long r0 = min(M, (long long)blockIdx.x * rs);
  return {r0, min(M, r0 + rs)};
}

// ---------------------------------------------------------------------------------------------------- forward
struct BnFold {
  const double* part;              // [S][2][C]: slice sums of x and x^2
  const float* gamma;
  const float* beta;
  float* run_mean;                 // updated by CTA 0
  float* run_var;
  double momentum, eps;
  double* stats;                   // [2][C] mean, invstd, written by CTA 0 for the backward; nullptr: not kept
};

// BN(x) = (x - mean) * scale + beta with mean and scale = gamma * invstd rounded once from double: torch's order (the
// subtraction first keeps a channel whose mean is far from 0 exact), and the same bits in the forward and in the
// backward's recomputation
__device__ inline void bn_affine(double mean, double invstd, float gamma, float& sc, float& sm) {
  sc = (float)((double)gamma * invstd);
  sm = (float)mean;
}
__device__ inline float bn_apply(float x, float sm, float sc, float beta) { return fmaf(x - sm, sc, beta); }

// the slice sums of `part` ([S][2][C]) in slice order, into tmp[2C] (C <= TRAIN_NT)
template <int C>
__device__ inline void sum_slices(const double* part, double* tmp) {
#pragma unroll
  for (int j = 0; j < (2 * C + TRAIN_NT - 1) / TRAIN_NT; ++j) {
    const int t = threadIdx.x + j * TRAIN_NT;
    if (t < 2 * C) {
      double s = 0.0;
      for (int z = 0; z < TRAIN_SLICES; ++z) s += part[z * 2 * C + t];
      tmp[t] = s;
    }
  }
  __syncthreads();
}

// the batch statistics of a BatchNorm's input -> its scale / mean / beta; CTA 0 also updates the running statistics
// (torch: running_var with the unbiased variance) and stores mean / invstd
template <int C>
__device__ void fold_bn(const BnFold& f, long long M, float* sc, float* sh, float* sb, double* tmp) {
  sum_slices<C>(f.part, tmp);
  const int c = threadIdx.x;
  if (c < C) {
    const double mean = tmp[c] / (double)M;
    const double var = fmax(tmp[C + c] / (double)M - mean * mean, 0.0);
    const double invstd = 1.0 / sqrt(var + f.eps);
    bn_affine(mean, invstd, f.gamma[c], sc[c], sh[c]);
    sb[c] = f.beta[c];
    if (blockIdx.x == 0) {
      if (f.stats != nullptr) {
        f.stats[c] = mean;
        f.stats[C + c] = invstd;
      }
      const double m = f.momentum;
      f.run_mean[c] = (float)((1.0 - m) * (double)f.run_mean[c] + m * mean);
      f.run_var[c] = (float)((1.0 - m) * (double)f.run_var[c] + m * var * (double)M / (double)(M - 1));
    }
  }
  __syncthreads();
}

// the row groups' per-channel (s1, s2) in group order -> this slice's partial part[blockIdx.x][2][C] (C <= TRAIN_NT)
template <int C, int G>
__device__ inline void write_slice_stats(double (*red)[2][C], int g, int c, double s1, double s2, double* part) {
  red[g][0][c] = s1;
  red[g][1][c] = s2;
  __syncthreads();
#pragma unroll
  for (int j = 0; j < (2 * C + TRAIN_NT - 1) / TRAIN_NT; ++j) {
    const int t = threadIdx.x + j * TRAIN_NT;
    if (t < 2 * C) {
      double s = 0.0;
      for (int q = 0; q < G; ++q) s += red[q][t / C][t % C];
      part[(long long)blockIdx.x * 2 * C + t] = s;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- backward
// BatchNorm backward from the gradient statistics, and gamma / beta's gradients (CTA 0)
struct BnGrad {
  const float* a; const double* stats; const float* gamma; const double* gpart;
  float* dgamma; float* dbeta;
};

// per channel, in double: k1 = gamma invstd, mg = Sigma g / M, mgx = Sigma g x_hat / M, mean, invstd.  The batch
// statistics' backward, da = k1 (g - mg - x_hat mgx), is formed in double with x_hat in double as in the statistics'
// sums, so that Sigma da -- the gradient of a bias in front of a BatchNorm, zero in exact arithmetic -- stays at
// double round-off
template <int C>
__device__ inline double bn_grad(float g, float a, int c, const double* k1, const double* mg, const double* mgx,
                                 const double* mean, const double* inv) {
  const double xh = ((double)a - mean[c]) * inv[c];
  return k1[c] * ((double)g - mg[c] - xh * mgx[c]);
}

template <int C>
__device__ void fold_bn_grad(const BnGrad& b, long long M, double* k1, double* mg, double* mgx, double* mean,
                             double* inv, double* tmp) {
  sum_slices<C>(b.gpart, tmp);
  const int c = threadIdx.x;
  if (c < C) {
    if (blockIdx.x == 0) {
      b.dbeta[c] = (float)tmp[c];
      b.dgamma[c] = (float)tmp[C + c];
    }
    k1[c] = (double)b.gamma[c] * b.stats[C + c];
    mg[c] = tmp[c] / (double)M;
    mgx[c] = tmp[C + c] / (double)M;
    mean[c] = b.stats[c];
    inv[c] = b.stats[C + c];
  }
  __syncthreads();
}

}  // namespace train
}  // namespace wekws
