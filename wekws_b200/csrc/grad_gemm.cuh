// The weight-gradient GEMM and the slice reduction of the FP32 training backwards (fsmn_grad.cu, gru_train.cu):
// every weight gradient dW = dY^T X is formed over FSMN_GRAD_SLICES fixed row slices, one thread summing a slice's
// rows in row order, and fsmn_grad_reduce_kernel adds the slices in slice order: no atomics, equal inputs give equal
// bits.  Internal linkage: each including file compiles its own copy.
#pragma once
#include "common.cuh"
#include "fsmn.h"

namespace wekws {

namespace {

// ---------------------------------------------------------------------------------------------------- GEMM
// C(i, j) = sum over kk in this block's slice of A(i, kk) B(kk, j), with A(i, kk) = A[i * sai + kk * sak] and
// B(kk, j) = Bm[kk * sbk + j * sbj] (optionally (Bm - bmean[j]) * bscale[j]: the CMVN of the features).
//   dX = dY W:     A = dY (M x N, sak = 1), B = W^T of the pack read as W (sbk = 1, sbj = Npad); C row-major (M x K),
//                  masked by mask[i][j] > 0 (the ReLU of the layer below) when mask != nullptr.
//   dW = dY^T X:   A = dY read transposed (sai = 1, sak = N), B = X (sbk = K, sbj = 1), blockIdx.z = row slice; C is the
//                  slice's partial [N][K]; with bias_out, the blocks of the first column tile also write the slice's
//                  column sums of dY (the bias gradient's partial).
constexpr int GB_M = 64, GB_N = 64, GB_K = 16, G_T = 256;

struct GemmArgs {
  const float* A; long long sai, sak;
  const float* B; long long sbk, sbj;
  const float* bmean; const float* bscale;       // per column j of B, or nullptr
  float* C; long long ldc, c_slice;              // C + z * c_slice
  const float* mask; long long ldm;              // nullptr: no mask
  float* bias_out; long long bias_slice;         // nullptr: no bias partial
  int I, J, K, kslice;                           // slice z covers kk in [z * kslice, min(K, (z + 1) * kslice))
};

__global__ void __launch_bounds__(G_T) fsmn_grad_gemm_kernel(const GemmArgs g) {
  __shared__ __align__(16) float As[GB_K][GB_M + 4];
  __shared__ __align__(16) float Bs[GB_K][GB_N + 4];
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int i0 = blockIdx.x * GB_M, j0 = blockIdx.y * GB_N;
  const int k_begin = blockIdx.z * g.kslice;
  const int k_end = min(g.K, k_begin + g.kslice);
  const bool a_kk_fast = g.sak == 1, b_j_fast = g.sbj == 1;
  const bool bias = g.bias_out != nullptr && blockIdx.y == 0 && tx == 0;
  float acc[4][4] = {}, bsum[4] = {};
  for (int k0 = k_begin; k0 < k_end; k0 += GB_K) {
#pragma unroll
    for (int q = 0; q < GB_M * GB_K / G_T; ++q) {
      const int e = tid + q * G_T;
      const int ii = a_kk_fast ? e / GB_K : e % GB_M, kk = a_kk_fast ? e % GB_K : e / GB_M;
      const int i = i0 + ii, k = k0 + kk;
      As[kk][ii] = i < g.I && k < k_end ? __ldg(g.A + i * g.sai + k * g.sak) : 0.f;
    }
#pragma unroll
    for (int q = 0; q < GB_N * GB_K / G_T; ++q) {
      const int e = tid + q * G_T;
      const int jj = b_j_fast ? e % GB_N : e / GB_K, kk = b_j_fast ? e / GB_N : e % GB_K;
      const int j = j0 + jj, k = k0 + kk;
      float v = 0.f;
      if (j < g.J && k < k_end) {
        v = __ldg(g.B + k * g.sbk + j * g.sbj);
        if (g.bmean != nullptr) v = (v - __ldg(g.bmean + j)) * __ldg(g.bscale + j);
      }
      Bs[kk][jj] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GB_K; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = fmaf(av[u], bv[v], acc[u][v]);
      if (bias) {
#pragma unroll
        for (int u = 0; u < 4; ++u) bsum[u] += av[u];
      }
    }
    __syncthreads();
  }
  float* C = g.C + blockIdx.z * g.c_slice;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int i = i0 + ty * 4 + u;
    if (i >= g.I) continue;
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int j = j0 + tx * 4 + v;
      if (j >= g.J) continue;
      float r = acc[u][v];
      if (g.mask != nullptr) r = __ldg(g.mask + i * g.ldm + j) > 0.f ? r : 0.f;   // torch's threshold_backward
      C[i * g.ldc + j] = r;
    }
    if (bias) g.bias_out[blockIdx.z * g.bias_slice + i] = bsum[u];
  }
}

int gemm(const GemmArgs& g, int slices, cudaStream_t st) {
  const dim3 grid((g.I + GB_M - 1) / GB_M, (g.J + GB_N - 1) / GB_N, slices);
  fsmn_grad_gemm_kernel<<<grid, G_T, 0, st>>>(g);
  return check_launch("fsmn_grad_gemm_kernel");
}

// ---------------------------------------------------------------------------------------------------- slice sums
struct ReduceJob {
  const float* part;   // [FSMN_GRAD_SLICES][n]
  float* out;          // [n]
  long long n;
};
struct ReduceArgs {
  int njobs;
  ReduceJob j[FSMN_MAX_PARAMS];
};

__global__ void fsmn_grad_reduce_kernel(const ReduceArgs a) {
  const ReduceJob& jb = a.j[blockIdx.y];
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < jb.n; e += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int z = 0; z < FSMN_GRAD_SLICES; ++z) s += __ldg(jb.part + z * jb.n + e);
    jb.out[e] = s;
  }
}

int reduce_slices(const ReduceArgs& r, cudaStream_t st) {
  long long most = 0;
  for (int i = 0; i < r.njobs; ++i) most = most > r.j[i].n ? most : r.j[i].n;
  const int bx = (int)((most + 255) / 256 < 128 ? (most + 255) / 256 : 128);
  fsmn_grad_reduce_kernel<<<dim3(bx, r.njobs), 256, 0, st>>>(r);
  return check_launch("fsmn_grad_reduce_kernel");
}

}  // namespace

}  // namespace wekws
