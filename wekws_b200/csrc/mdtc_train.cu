// MDTC training (wekws/utils/executor.py Executor.train through wekws/model/mdtc.py): the training-mode forward, with
// every BatchNorm normalising by the statistics of the batch and updating its running statistics, and the backward to
// every parameter of the reference's MDTC model with the per-frame linear classifier.
//
// FP32 FMA throughout (the 64 x 64 and 32 x 32 GEMMs of mdtc.yaml / mdtc_small.yaml).  Activations are channel-last
// (M = B * T rows of C floats), every frame a row, padding included, as torch's BatchNorm1d takes them.  Every launch
// runs MDTC_TRAIN_SLICES CTAs, CTA z owning the fixed row slice z.  A batch statistic (Sigma x, Sigma x^2 of the
// forward; Sigma g, Sigma g x_hat of the backward) is formed per slice in double, the row groups of a CTA added in
// group order, and every CTA of the next launch adds the slices in slice order in its prologue.  Weight gradients are
// per-slice partials in double, added in slice order by one final launch that rounds once.  No atomics: equal inputs give equal bits.
//
// Per block (input x: the preprocessing output for the preprocessor, else the previous block's output y):
//   a0 = depthwise_dilated_causal(x) + b0          dw kernel (also: x itself, computed on load, is stored once)
//   a1 = Wp BN0(a0) + bp                           pw kernel
//   a2 = W2 relu(BN1(a1)) + b2                     pw kernel
//   y  = relu(BN2(a2) + x)                         computed on load by the next block's dw kernel / the final kernel
// The saved buffer keeps only the pre-BN tensors, the block inputs / outputs and the stack sum; x_hat is recomputed.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "mdtc_train.h"
#include "train_common.cuh"

namespace wekws {

namespace {

using namespace train;
constexpr int S = MDTC_TRAIN_SLICES;
constexpr int NT = TRAIN_NT;
static_assert(S == TRAIN_SLICES, "the MDTC slices are the shared scheme's");

// ---------------------------------------------------------------------------------------------------- forward
// preprocessing Linear(idim, C) + ReLU of the CMVN-normalised features
struct PreArgs {
  const float* x; const float* mean; const float* istd; int norm_var;
  const float* W; const float* b; float* h0;
  long long M; int idim;
};

template <int C>
__global__ void __launch_bounds__(NT) mdtc_train_pre_kernel(const PreArgs a) {
  constexpr int G = NT / C, RC = 16;
  __shared__ float Wt[MDTC_TRAIN_MAX_IDIM * C];
  __shared__ float xs[RC * MDTC_TRAIN_MAX_IDIM];
  const int idim = a.idim;
  for (int e = threadIdx.x; e < idim * C; e += NT) Wt[(e % idim) * C + e / idim] = a.W[e];
  const Rows sl = slice_rows(a.M);
  const int c = threadIdx.x % C, g = threadIdx.x / C;
  const float bias = a.b[c];
  for (long long q0 = sl.r0; q0 < sl.r1; q0 += RC) {
    const int nr = (int)min((long long)RC, sl.r1 - q0);
    __syncthreads();
    for (int e = threadIdx.x; e < nr * idim; e += NT) {
      float v = a.x[q0 * idim + e];
      if (a.mean != nullptr) {                       // wekws/model/cmvn.py: x - mean, then * istd if norm_var
        const int i = e % idim;
        v = v - a.mean[i];
        if (a.norm_var) v = v * a.istd[i];
      }
      xs[e] = v;
    }
    __syncthreads();
    for (int r = g; r < nr; r += G) {
      float acc = bias;
      for (int i = 0; i < idim; ++i) acc = fmaf(xs[r * idim + i], Wt[i * C + c], acc);
      a.h0[(q0 + r) * C + c] = fmaxf(acc, 0.f);
    }
  }
}

// depthwise dilated causal conv + bias of the block input x, with x computed on load: x = res for the preprocessor,
// else relu(BN2(a2) + res) of the previous block (stored once at y_out, and added to the stack sum at a stack end).
// Also the block's slice of the out_cache (the last `pad` input frames, zeros before frame 0) and a0's slice stats.
struct DwArgs {
  const float* a2; const float* res; BnFold f2;      // a2 == nullptr: x = res
  float* y_out; float* ssum; int ssum_mode;          // ssum_mode: 0 none, 1 ssum = x, 2 ssum += x
  const float* w; const float* bias; float* a0; double* part;
  float* cache; int cache_off, pad, ptot;
  long long M; int T, K, dil;
};

template <int C>
__global__ void __launch_bounds__(NT) mdtc_train_dw_kernel(const DwArgs a) {
  constexpr int G = NT / C;
  __shared__ float sc[C], sh[C], sb[C];
  __shared__ double tmp[2 * C];
  __shared__ double red[G][2][C];
  const bool fused = a.a2 != nullptr;
  if (fused) fold_bn<C>(a.f2, a.M, sc, sh, sb, tmp);
  const Rows sl = slice_rows(a.M);
  const int c = threadIdx.x % C, g = threadIdx.x / C;
  const float s2 = fused ? sc[c] : 0.f, h2 = fused ? sh[c] : 0.f, b2 = fused ? sb[c] : 0.f;
  float w[MDTC_TRAIN_MAX_K];
#pragma unroll
  for (int k = 0; k < MDTC_TRAIN_MAX_K; ++k) w[k] = k < a.K ? a.w[c * a.K + k] : 0.f;
  const float bias = a.bias[c];
  double s1 = 0.0, sq = 0.0;
  for (long long r = sl.r0 + g; r < sl.r1; r += G) {
    const int t = (int)(r % a.T);
    const long long base = r - t;
    float acc = bias, cur = 0.f;
#pragma unroll
    for (int k = 0; k < MDTC_TRAIN_MAX_K; ++k) {
      if (k >= a.K) break;
      const int u = t - (a.K - 1 - k) * a.dil;
      float v = 0.f;
      if (u >= 0) {
        const long long i = (base + u) * C + c;
        v = fused ? fmaxf(bn_apply(a.a2[i], h2, s2, b2) + a.res[i], 0.f) : a.res[i];
      }
      acc = fmaf(w[k], v, acc);
      cur = v;                                      // the last tap is frame t itself
    }
    a.a0[r * C + c] = acc;
    s1 += (double)acc;
    sq += (double)acc * (double)acc;
    if (a.y_out != nullptr) a.y_out[r * C + c] = cur;
    if (a.ssum_mode == 1) a.ssum[r * C + c] = cur;
    else if (a.ssum_mode == 2) a.ssum[r * C + c] += cur;
    float* cache = a.cache + ((base / a.T) * C + c) * a.ptot + a.cache_off;
    const int j = a.pad - a.T + t;                  // mdtc.py: the last `pad` frames of [zeros(pad) | x]
    if (j >= 0) cache[j] = cur;
    if (t == a.T - 1)
      for (int z = 0; z < a.pad - a.T; ++z) cache[z] = 0.f;
  }
  write_slice_stats<C, G>(red, g, c, s1, sq, a.part);
}

// a = W n + bias over the channels, n = BN(in) (then ReLU when relu_in), with a's slice stats
struct PwArgs {
  const float* in; BnFold f; int relu_in;
  const float* W; const float* bias; float* out; double* part;
  long long M;
};

template <int C>
__global__ void __launch_bounds__(NT) mdtc_train_pw_kernel(const PwArgs a) {
  constexpr int RC = 64, CPT = C / 16;
  static_assert(C * (RC + 4) * 4 >= 16 * 2 * C * 8, "the statistics reuse xs");
  __shared__ __align__(16) float xs[C][RC + 4];      // n^T: [channel][row]
  __shared__ __align__(16) float Wt[C][C];           // W^T: [in][out]
  __shared__ float sc[C], sh[C], sb[C];
  __shared__ double tmp[2 * C];
  fold_bn<C>(a.f, a.M, sc, sh, sb, tmp);
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  for (int e = tid; e < C * C; e += NT) Wt[e % C][e / C] = a.W[e];
  float bias[CPT];
#pragma unroll
  for (int v = 0; v < CPT; ++v) bias[v] = a.bias[tx * CPT + v];
  double s1[CPT], sq[CPT];
#pragma unroll
  for (int v = 0; v < CPT; ++v) s1[v] = sq[v] = 0.0;
  const Rows sl = slice_rows(a.M);
  for (long long q0 = sl.r0; q0 < sl.r1; q0 += RC) {
    const int nr = (int)min((long long)RC, sl.r1 - q0);
    __syncthreads();
    for (int e = tid; e < RC * C; e += NT) {
      const int r = e / C, i = e % C;
      float v = 0.f;
      if (r < nr) {
        v = bn_apply(a.in[(q0 + r) * C + i], sh[i], sc[i], sb[i]);
        if (a.relu_in) v = fmaxf(v, 0.f);
      }
      xs[i][r] = v;
    }
    __syncthreads();
    float acc[4][CPT];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < CPT; ++v) acc[u][v] = bias[v];
#pragma unroll 8
    for (int i = 0; i < C; ++i) {
      const float4 x4 = *reinterpret_cast<const float4*>(&xs[i][ty * 4]);
      const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
      float wv[CPT];
#pragma unroll
      for (int v = 0; v < CPT; ++v) wv[v] = Wt[i][tx * CPT + v];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < CPT; ++v) acc[u][v] = fmaf(wv[v], xv[u], acc[u][v]);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int r = ty * 4 + u;
      if (r >= nr) continue;
#pragma unroll
      for (int v = 0; v < CPT; ++v) {
        a.out[(q0 + r) * C + tx * CPT + v] = acc[u][v];
        s1[v] += (double)acc[u][v];
        sq[v] += (double)acc[u][v] * (double)acc[u][v];
      }
    }
  }
  __syncthreads();
  auto red = reinterpret_cast<double (*)[2][C]>(&xs[0][0]);
#pragma unroll
  for (int v = 0; v < CPT; ++v) {
    red[ty][0][tx * CPT + v] = s1[v];
    red[ty][1][tx * CPT + v] = sq[v];
  }
  __syncthreads();
  if (tid < 2 * C) {
    double s = 0.0;
    for (int q = 0; q < 16; ++q) s += red[q][tid / C][tid % C];
    a.part[(long long)blockIdx.x * 2 * C + tid] = s;
  }
}

// the last block's output y = relu(BN2(a2) + res), the stack sum, the classifier and the activation
struct FinalArgs {
  const float* a2; const float* res; BnFold f2;
  float* y_out; float* ssum; int ssum_mode;
  const float* Wc; const float* bc; float* out; int O, act;
  long long M;
};

__device__ inline float classify(const float* s, const float* Wc, const float* bc, int o, int C, int act) {
  float z = bc[o];
  for (int c = 0; c < C; ++c) z = fmaf(Wc[o * C + c], s[c], z);
  return act ? 1.f / (1.f + expf(-z)) : z;
}

template <int C>
__global__ void __launch_bounds__(NT) mdtc_train_final_kernel(const FinalArgs a) {
  constexpr int G = NT / C, RC = 32;
  __shared__ float sc[C], sh[C], sb[C];
  __shared__ double tmp[2 * C];
  __shared__ float ss[RC][C + 1];
  fold_bn<C>(a.f2, a.M, sc, sh, sb, tmp);
  const Rows sl = slice_rows(a.M);
  const int c = threadIdx.x % C, g = threadIdx.x / C;
  for (long long q0 = sl.r0; q0 < sl.r1; q0 += RC) {
    const int nr = (int)min((long long)RC, sl.r1 - q0);
    __syncthreads();
    for (int r = g; r < nr; r += G) {
      const long long i = (q0 + r) * C + c;
      const float y = fmaxf(bn_apply(a.a2[i], sh[c], sc[c], sb[c]) + a.res[i], 0.f);
      if (a.y_out != nullptr) a.y_out[i] = y;
      const float s = a.ssum_mode == 1 ? y : a.ssum[i] + y;
      a.ssum[i] = s;
      ss[r][c] = s;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < nr * a.O; e += NT) {
      const int r = e / a.O, o = e % a.O;
      a.out[(q0 + r) * a.O + o] = classify(ss[r], a.Wc, a.bc, o, C, a.act);
    }
  }
}

// ---------------------------------------------------------------------------------------------------- backward
// classifier: dz = g * sigmoid'(z) (z recomputed as the forward did); ds = dz Wc; dWc, dbc slice partials
struct ClsBwdArgs {
  const float* g; const float* ssum; const float* Wc; const float* bc; int O, act;
  float* ds; double* dW_part; double* db_part;
  long long M;
};

template <int C>
__global__ void __launch_bounds__(NT) mdtc_train_cls_bwd_kernel(const ClsBwdArgs a) {
  constexpr int RC = 32, J = (MDTC_TRAIN_MAX_ODIM * C + NT - 1) / NT;
  __shared__ float ss[RC][C + 1];
  __shared__ float dz[RC][MDTC_TRAIN_MAX_ODIM + 1];
  const int tid = threadIdx.x, O = a.O;
  double acc[J];
#pragma unroll
  for (int j = 0; j < J; ++j) acc[j] = 0.0;
  double accb = 0.0;
  const Rows sl = slice_rows(a.M);
  for (long long q0 = sl.r0; q0 < sl.r1; q0 += RC) {
    const int nr = (int)min((long long)RC, sl.r1 - q0);
    __syncthreads();
    for (int e = tid; e < RC * C; e += NT) {
      const int r = e / C, c = e % C;
      ss[r][c] = r < nr ? a.ssum[(q0 + r) * C + c] : 0.f;
    }
    __syncthreads();
    for (int e = tid; e < RC * O; e += NT) {
      const int r = e / O, o = e % O;
      float d = 0.f;
      if (r < nr) {
        d = a.g[(q0 + r) * O + o];
        if (a.act) {                                 // g * (1 - y) * y, y = sigmoid(z) with z in double
          double z = a.bc[o];
          for (int c = 0; c < C; ++c) z = fma((double)a.Wc[o * C + c], (double)ss[r][c], z);
          const double y = 1.0 / (1.0 + exp(-z));
          d = (float)((double)d * (1.0 - y) * y);
        }
      }
      dz[r][o] = d;
    }
    __syncthreads();
    for (int e = tid; e < nr * C; e += NT) {
      const int r = e / C, c = e % C;
      float s = 0.f;
      for (int o = 0; o < O; ++o) s = fmaf(dz[r][o], a.Wc[o * C + c], s);
      a.ds[(q0 + r) * C + c] = s;
    }
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int p = tid + j * NT;
      if (p < O * C) {
        const int o = p / C, c = p % C;
        for (int r = 0; r < nr; ++r) acc[j] = fma((double)dz[r][o], (double)ss[r][c], acc[j]);
      }
    }
    if (tid < O)
      for (int r = 0; r < nr; ++r) accb += dz[r][tid];
  }
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int p = tid + j * NT;
    if (p < O * C) a.dW_part[(long long)blockIdx.x * O * C + p] = acc[j];
  }
  if (tid < O) a.db_part[(long long)blockIdx.x * O + tid] = accb;
}

// BN2's gradient statistics: g = dy * [y > 0] (the block's closing ReLU), Sigma g and Sigma g x_hat per slice
struct GStatArgs {
  const float* dy; const float* y; const float* a; const double* stats; double* part;
  long long M;
};

template <int C>
__global__ void __launch_bounds__(NT) mdtc_train_gstat_kernel(const GStatArgs a) {
  constexpr int G = NT / C;
  __shared__ double red[G][2][C];
  const int c = threadIdx.x % C, g = threadIdx.x / C;
  const double mean = a.stats[c], inv = a.stats[C + c];
  double s1 = 0.0, s2 = 0.0;
  const Rows sl = slice_rows(a.M);
  for (long long r = sl.r0 + g; r < sl.r1; r += G) {
    const long long i = r * C + c;
    const float gv = a.y[i] > 0.f ? a.dy[i] : 0.f;
    s1 += (double)gv;
    s2 += (double)gv * (((double)a.a[i] - mean) * inv);
  }
  write_slice_stats<C, G>(red, g, c, s1, s2, a.part);
}

// The backward of a = W n + bias, n = [relu](BN_in(a_in)), from the gradient into BN_out(a) (g = up [* (ymask > 0)]):
// da = BN_out backward; dn = da W, masked by [n > 0] when relu_in, stored with its slice stats against BN_in's x_hat;
// dW = da^T n and db = Sigma da as slice partials.
struct PwBwdArgs {
  const float* up; const float* ymask; BnGrad bo;
  const float* W; const float* a_in; const double* st_in; const float* gamma_in; const float* beta_in; int relu_in;
  double* dW_part; double* db_part; float* dn; double* part;
  long long M;
};

template <int C>
__global__ void __launch_bounds__(NT) mdtc_train_pw_bwd_kernel(const PwBwdArgs a) {
  constexpr int RC = 32, RPT = RC / 16, CPT = C / 16, LD = C + 4;
  static_assert(2 * RC * LD * 4 >= 16 * 2 * C * 8, "the statistics reuse DA / N");
  __shared__ __align__(16) float buf[2 * RC * LD];
  float (*DA)[LD] = reinterpret_cast<float (*)[LD]>(buf);              // da [row][out channel]
  float (*N)[LD] = reinterpret_cast<float (*)[LD]>(buf + RC * LD);     // n  [row][in channel]
  __shared__ __align__(16) float Ws[C][C];                             // W  [out][in]
  __shared__ double k1[C], mg[C], mgx[C], mo[C], io[C], mi[C], ii[C];
  __shared__ float sci[C], shi[C], sbi[C];
  __shared__ double tmp[2 * C];
  fold_bn_grad<C>(a.bo, a.M, k1, mg, mgx, mo, io, tmp);
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  if (tid < C) {
    bn_affine(a.st_in[tid], a.st_in[C + tid], a.gamma_in[tid], sci[tid], shi[tid]);
    sbi[tid] = a.beta_in[tid];
    mi[tid] = a.st_in[tid];
    ii[tid] = a.st_in[C + tid];
  }
  for (int e = tid; e < C * C; e += NT) Ws[e / C][e % C] = a.W[e];
  double accW[CPT][CPT];
#pragma unroll
  for (int u = 0; u < CPT; ++u)
#pragma unroll
    for (int v = 0; v < CPT; ++v) accW[u][v] = 0.0;
  double pb = 0.0;                                     // Sigma da of channel tid % C over this thread's rows
  double s1[CPT], s2[CPT];
#pragma unroll
  for (int v = 0; v < CPT; ++v) s1[v] = s2[v] = 0.0;
  const Rows sl = slice_rows(a.M);
  for (long long q0 = sl.r0; q0 < sl.r1; q0 += RC) {
    const int nr = (int)min((long long)RC, sl.r1 - q0);
    __syncthreads();
    for (int e = tid; e < RC * C; e += NT) {
      const int r = e / C, c = e % C;
      float da = 0.f, n = 0.f;
      if (r < nr) {
        const long long i = (q0 + r) * C + c;
        float gv = a.up[i];
        if (a.ymask != nullptr && !(a.ymask[i] > 0.f)) gv = 0.f;
        const double dd = bn_grad<C>(gv, a.bo.a[i], c, k1, mg, mgx, mo, io);
        pb += dd;
        da = (float)dd;
        n = bn_apply(a.a_in[i], shi[c], sci[c], sbi[c]);
        if (a.relu_in) n = fmaxf(n, 0.f);
      }
      DA[r][c] = da;
      N[r][c] = n;
    }
    __syncthreads();
    // dn = da W
    float acc[RPT][CPT];
#pragma unroll
    for (int u = 0; u < RPT; ++u)
#pragma unroll
      for (int v = 0; v < CPT; ++v) acc[u][v] = 0.f;
#pragma unroll 8
    for (int o = 0; o < C; ++o) {
      float wv[CPT];
#pragma unroll
      for (int v = 0; v < CPT; ++v) wv[v] = Ws[o][tx * CPT + v];
#pragma unroll
      for (int u = 0; u < RPT; ++u) {
        const float d = DA[ty * RPT + u][o];
#pragma unroll
        for (int v = 0; v < CPT; ++v) acc[u][v] = fmaf(d, wv[v], acc[u][v]);
      }
    }
#pragma unroll
    for (int u = 0; u < RPT; ++u) {
      const int r = ty * RPT + u;
      if (r >= nr) continue;
#pragma unroll
      for (int v = 0; v < CPT; ++v) {
        const int c = tx * CPT + v;
        const long long i = (q0 + r) * C + c;
        float d = acc[u][v];
        if (a.relu_in && !(N[r][c] > 0.f)) d = 0.f;   // torch's threshold_backward
        a.dn[i] = d;
        s1[v] += (double)d;
        s2[v] += (double)d * (((double)a.a_in[i] - mi[c]) * ii[c]);
      }
    }
    // dW[o][c] += da[r][o] n[r][c] for o in ty's, c in tx's columns
    for (int r = 0; r < nr; ++r) {
      float dv[CPT], nv[CPT];
#pragma unroll
      for (int u = 0; u < CPT; ++u) dv[u] = DA[r][ty * CPT + u];
#pragma unroll
      for (int v = 0; v < CPT; ++v) nv[v] = N[r][tx * CPT + v];
#pragma unroll
      for (int u = 0; u < CPT; ++u)
#pragma unroll
        for (int v = 0; v < CPT; ++v) accW[u][v] = fma((double)dv[u], (double)nv[v], accW[u][v]);
    }
  }
  double* dW = a.dW_part + (long long)blockIdx.x * C * C;
#pragma unroll
  for (int u = 0; u < CPT; ++u)
#pragma unroll
    for (int v = 0; v < CPT; ++v) dW[(ty * CPT + u) * C + tx * CPT + v] = accW[u][v];
  __syncthreads();
  auto redb = reinterpret_cast<double (*)[C]>(buf);                    // the bias partial: thread groups in order
  redb[tid / C][tid % C] = pb;
  __syncthreads();
  if (tid < C) {
    double sb = 0.0;
    for (int q = 0; q < NT / C; ++q) sb += redb[q][tid];
    a.db_part[(long long)blockIdx.x * C + tid] = sb;
  }
  __syncthreads();
  auto red = reinterpret_cast<double (*)[2][C]>(buf);
#pragma unroll
  for (int v = 0; v < CPT; ++v) {
    red[ty][0][tx * CPT + v] = s1[v];
    red[ty][1][tx * CPT + v] = s2[v];
  }
  __syncthreads();
  if (tid < 2 * C) {
    double s = 0.0;
    for (int q = 0; q < 16; ++q) s += red[q][tid / C][tid % C];
    a.part[(long long)blockIdx.x * 2 * C + tid] = s;
  }
}

// BN0 backward, then the depthwise conv's: d_in (within each utterance) plus the residual dy * [y > 0] (plus the stack
// sum's gradient ds when the input is a stack's output; times [in > 0] for the preprocessing ReLU of block 0); tap
// and bias gradients as slice partials [C][K], [C].
struct DwBwdArgs {
  const float* dn0; BnGrad b0;
  const float* w; const float* in;
  const float* dy; const float* y; const float* ds; int mask_in;
  float* d_in; double* dw_part; double* db_part;
  long long M; int T, K, dil;
};

template <int C>
__global__ void __launch_bounds__(NT) mdtc_train_dw_bwd_kernel(const DwBwdArgs a) {
  constexpr int G = NT / C, KP = MDTC_TRAIN_MAX_K + 1;
  __shared__ double k1[C], mg[C], mgx[C], m0[C], i0[C];
  __shared__ double tmp[2 * C];
  __shared__ double red[G][KP][C];
  fold_bn_grad<C>(a.b0, a.M, k1, mg, mgx, m0, i0, tmp);
  const int c = threadIdx.x % C, g = threadIdx.x / C;
  float w[MDTC_TRAIN_MAX_K];
  double acc[KP];
#pragma unroll
  for (int k = 0; k < MDTC_TRAIN_MAX_K; ++k) w[k] = k < a.K ? a.w[c * a.K + k] : 0.f;
#pragma unroll
  for (int k = 0; k < KP; ++k) acc[k] = 0.0;
  auto da = [&](long long row) {
    const long long i = row * C + c;
    return bn_grad<C>(a.dn0[i], a.b0.a[i], c, k1, mg, mgx, m0, i0);
  };
  const Rows sl = slice_rows(a.M);
  for (long long r = sl.r0 + g; r < sl.r1; r += G) {
    const int t = (int)(r % a.T);
    const long long base = r - t, i = r * C + c;
    const double dself = da(r);
    float d = 0.f;
#pragma unroll
    for (int k = 0; k < MDTC_TRAIN_MAX_K; ++k) {
      if (k >= a.K) break;
      const int sh = (a.K - 1 - k) * a.dil;
      if (t + sh < a.T) d = fmaf(w[k], (float)(sh == 0 ? dself : da(base + t + sh)), d);   // output t + sh read x[t]
      if (t - sh >= 0) acc[k] = fma(dself, (double)a.in[(base + t - sh) * C + c], acc[k]);
    }
    acc[MDTC_TRAIN_MAX_K] += dself;
    if (a.y[i] > 0.f) d += a.dy[i];                  // the residual through the block's closing ReLU
    if (a.ds != nullptr) d += a.ds[i];
    if (a.mask_in && !(a.in[i] > 0.f)) d = 0.f;
    a.d_in[i] = d;
  }
#pragma unroll
  for (int k = 0; k < KP; ++k) red[g][k][c] = acc[k];
  __syncthreads();
  for (int e = threadIdx.x; e < (a.K + 1) * C; e += NT) {
    const int k = e / C, cc = e % C, kk = k < a.K ? k : MDTC_TRAIN_MAX_K;
    double s = 0.0;
    for (int q = 0; q < G; ++q) s += red[q][kk][cc];
    if (k < a.K) a.dw_part[(long long)blockIdx.x * C * a.K + cc * a.K + k] = s;
    else a.db_part[(long long)blockIdx.x * C + cc] = s;
  }
}

// the preprocessing Linear's dW = d^T CMVN(x), db = Sigma d as slice partials
struct PreBwdArgs {
  const float* d; const float* x; const float* mean; const float* istd; int norm_var;
  double* dW_part; double* db_part;
  long long M; int idim;
};

template <int C>
__global__ void __maxnreg__(128) mdtc_train_pre_bwd_kernel(const PreBwdArgs a) {
  constexpr int RC = 16, J = (MDTC_TRAIN_MAX_IDIM * C + NT - 1) / NT;
  __shared__ float ds[RC][C];
  __shared__ float xs[RC][MDTC_TRAIN_MAX_IDIM];
  const int tid = threadIdx.x, idim = a.idim, n = C * idim;
  double acc[J];
#pragma unroll
  for (int j = 0; j < J; ++j) acc[j] = 0.0;
  double accb = 0.0;
  const Rows sl = slice_rows(a.M);
  for (long long q0 = sl.r0; q0 < sl.r1; q0 += RC) {
    const int nr = (int)min((long long)RC, sl.r1 - q0);
    __syncthreads();
    for (int e = tid; e < nr * C; e += NT) ds[e / C][e % C] = a.d[q0 * C + e];
    for (int e = tid; e < nr * idim; e += NT) {
      const int i = e % idim;
      float v = a.x[q0 * idim + e];
      if (a.mean != nullptr) {
        v = v - a.mean[i];
        if (a.norm_var) v = v * a.istd[i];
      }
      xs[e / idim][i] = v;
    }
    __syncthreads();
    for (int r = 0; r < nr; ++r) {
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int p = tid + j * NT;
        if (p < n) acc[j] = fma((double)ds[r][p / idim], (double)xs[r][p % idim], acc[j]);
      }
      if (tid < C) accb += ds[r][tid];
    }
  }
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int p = tid + j * NT;
    if (p < n) a.dW_part[(long long)blockIdx.x * n + p] = acc[j];
  }
  if (tid < C) a.db_part[(long long)blockIdx.x * C + tid] = accb;
}

// every weight / bias gradient: its slice partials added in slice order
constexpr int MAX_JOBS = 4 + 6 * MDTC_TRAIN_MAX_BLOCKS;   // 3.7 KB of kernel parameters
struct ReduceJob {
  const double* part;    // [S][n]
  float* out;
  int n;
};
struct ReduceArgs {
  ReduceJob j[MAX_JOBS];
};

__global__ void mdtc_train_reduce_kernel(const ReduceArgs a) {
  const ReduceJob& jb = a.j[blockIdx.y];
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < jb.n; e += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int z = 0; z < S; ++z) s += jb.part[(long long)z * jb.n + e];
    jb.out[e] = (float)s;
  }
}

// ---------------------------------------------------------------------------------------------------- host side
// the parameters of block b (index into the named_parameters order)
inline int pidx(int b, int k) { return 2 + 12 * b + k; }
inline int bn_index(int b, int which) { return 3 * b + which; }     // which: 0 conv1.bn, 1 bn1, 2 bn2

// the sliced gradients in parameter order: preprocessing W, b; per block dw W, b, pointwise W, b, conv2 W, b; classifier
std::vector<long long> sliced_sizes(const MdtcTrainDims& d) {
  const long long C = d.C;
  std::vector<long long> n = {C * d.idim, C};
  for (int b = 0; b < d.L; ++b) {
    const long long blk[6] = {C * d.K, C, C * C, C, C * C, C};
    n.insert(n.end(), blk, blk + 6);
  }
  n.push_back((long long)d.odim * C);
  n.push_back(d.odim);
  return n;
}

long long sliced_total(const MdtcTrainDims& d) {
  long long s = 0;
  for (long long v : sliced_sizes(d)) s += v;
  return s;
}

template <int C>
int forward_t(const MdtcTrainDims& d, const float* feats, const float* const* P, const float* cmvn_mean,
              const float* cmvn_istd, float* const* running, const double* bn, float* out, float* out_cache,
              float* saved, void* workspace, int B, int T, cudaStream_t st) {
  const long long M = (long long)B * T, MC = M * C;
  const int L = d.L;
  double* part[3];
  double* w8 = (double*)workspace;
  for (int i = 0; i < 3; ++i) part[i] = w8 + (long long)i * S * 2 * C;
  float* ws = (float*)(w8 + 3LL * S * 2 * C);
  // where each activation lives: every block's own in the saved buffer (layout: [3 L BatchNorms' (mean, invstd) x C
  // doubles] [h0] [per block a0, a1, a2, y] [stack sum]), or rings in the workspace (h0 and the block outputs share two
  // slots: block b's dw kernel reads y(b - 2) and writes y(b - 1))
  double* stats = saved ? (double*)saved : nullptr;
  float* act = saved ? saved + 12LL * L * C : ws;
  auto h0 = act;
  auto a0 = [&](int b) { return saved ? act + MC * (1 + 4LL * b) : act + 2 * MC; };
  auto a1 = [&](int b) { return saved ? act + MC * (2 + 4LL * b) : act + 3 * MC; };
  auto a2 = [&](int b) { return saved ? act + MC * (3 + 4LL * b) : act + 4 * MC; };
  auto y = [&](int b) { return b < 0 ? h0 : saved ? act + MC * (4 + 4LL * b) : act + MC * ((b + 1) % 2); };
  float* ssum = saved ? act + MC * (1 + 4LL * L) : act + 5 * MC;
  auto fold = [&](int b, int which, const double* p) {
    const int k = bn_index(b, which);
    BnFold f{};
    f.part = p;
    f.gamma = P[pidx(b, which == 0 ? 2 : which == 1 ? 6 : 10)];
    f.beta = P[pidx(b, which == 0 ? 3 : which == 1 ? 7 : 11)];
    f.run_mean = running[2 * k];
    f.run_var = running[2 * k + 1];
    f.momentum = bn[2 * k];
    f.eps = bn[2 * k + 1];
    f.stats = stats ? stats + (long long)k * 2 * C : nullptr;
    return f;
  };
  auto ssum_mode = [&](int b) { return !mdtc_stack_end(b, d.stack_size) ? 0 : b == d.stack_size ? 1 : 2; };
  int rc;
  {
    PreArgs p{};
    p.x = feats; p.mean = cmvn_mean; p.istd = cmvn_istd; p.norm_var = d.norm_var;
    p.W = P[0]; p.b = P[1]; p.h0 = h0; p.M = M; p.idim = d.idim;
    mdtc_train_pre_kernel<C><<<S, NT, 0, st>>>(p);
    if ((rc = check_launch("mdtc_train_pre_kernel"))) return rc;
  }
  for (int b = 0; b < L; ++b) {
    DwArgs a{};
    if (b > 0) {
      a.a2 = a2(b - 1); a.f2 = fold(b - 1, 2, part[2]);
      a.y_out = y(b - 1); a.ssum = ssum; a.ssum_mode = ssum_mode(b - 1);
    }
    a.res = y(b - 2);
    a.w = P[pidx(b, 0)]; a.bias = P[pidx(b, 1)]; a.a0 = a0(b); a.part = part[0];
    a.cache = out_cache; a.cache_off = d.coff[b]; a.pad = d.dil[b] * (d.K - 1); a.ptot = d.pad_total;
    a.M = M; a.T = T; a.K = d.K; a.dil = d.dil[b];
    mdtc_train_dw_kernel<C><<<S, NT, 0, st>>>(a);
    if ((rc = check_launch("mdtc_train_dw_kernel"))) return rc;
    for (int which = 0; which < 2; ++which) {
      PwArgs q{};
      q.in = which == 0 ? a0(b) : a1(b);
      q.f = fold(b, which, part[which]);
      q.relu_in = which;
      q.W = P[pidx(b, which == 0 ? 4 : 8)]; q.bias = P[pidx(b, which == 0 ? 5 : 9)];
      q.out = which == 0 ? a1(b) : a2(b);
      q.part = part[which + 1];
      q.M = M;
      mdtc_train_pw_kernel<C><<<S, NT, 0, st>>>(q);
      if ((rc = check_launch("mdtc_train_pw_kernel"))) return rc;
    }
  }
  FinalArgs f{};
  f.a2 = a2(L - 1); f.res = y(L - 2); f.f2 = fold(L - 1, 2, part[2]);
  f.y_out = saved ? y(L - 1) : nullptr; f.ssum = ssum; f.ssum_mode = ssum_mode(L - 1);
  if (d.odim > 0) { f.Wc = P[2 + 12 * L]; f.bc = P[3 + 12 * L]; }     // odim 0: the stack sum is the output
  f.out = out; f.O = d.odim; f.act = d.act; f.M = M;
  mdtc_train_final_kernel<C><<<S, NT, 0, st>>>(f);
  return check_launch("mdtc_train_final_kernel");
}

template <int C>
int backward_t(const MdtcTrainDims& d, const float* feats, const float* const* P, const float* cmvn_mean,
               const float* cmvn_istd, const float* saved, const float* grad_out, int B, int T, float* const* grads,
               void* workspace, cudaStream_t st) {
  const long long M = (long long)B * T, MC = M * C;
  const int L = d.L;
  const double* stats = (const double*)saved;
  const float* act = saved + 12LL * L * C;
  const float* h0 = act;
  auto a0 = [&](int b) { return act + MC * (1 + 4LL * b); };
  auto a1 = [&](int b) { return act + MC * (2 + 4LL * b); };
  auto a2 = [&](int b) { return act + MC * (3 + 4LL * b); };
  auto y = [&](int b) { return b < 0 ? h0 : act + MC * (4 + 4LL * b); };
  const float* ssum = act + MC * (1 + 4LL * L);
  auto bstats = [&](int b, int which) { return stats + (long long)bn_index(b, which) * 2 * C; };
  // workspace: [gradient statistics x 2][ds][dy x 2][t1][t2][slice partials of every sliced gradient, in order, as
  // doubles]
  double* gpart[2] = {(double*)workspace, (double*)workspace + 2LL * S * C};
  float* ds_ws = (float*)((double*)workspace + 4LL * S * C);
  const float* ds = d.odim > 0 ? ds_ws : grad_out;            // odim 0: grad_out is the stack sum's gradient
  float* dyr[2] = {ds_ws + MC, ds_ws + 2 * MC};
  float* t1 = ds_ws + 3 * MC;
  float* t2 = ds_ws + 4 * MC;
  const std::vector<long long> sizes = sliced_sizes(d);
  std::vector<double*> part(sizes.size());
  double* w = (double*)(ds_ws + 5 * MC);
  for (size_t i = 0; i < sizes.size(); ++i) { part[i] = w; w += S * sizes[i]; }
  auto dy = [&](int b) -> const float* { return b == L - 1 ? ds : dyr[b % 2]; };   // the last block is a stack end
  auto bng = [&](int b, int which, const float* a, const double* gp) {
    BnGrad g{};
    g.a = a; g.stats = bstats(b, which); g.gamma = P[pidx(b, which == 0 ? 2 : which == 1 ? 6 : 10)]; g.gpart = gp;
    g.dgamma = grads[pidx(b, which == 0 ? 2 : which == 1 ? 6 : 10)];
    g.dbeta = grads[pidx(b, which == 0 ? 3 : which == 1 ? 7 : 11)];
    return g;
  };
  int rc;
  if (d.odim > 0) {
    ClsBwdArgs c{};
    c.g = grad_out; c.ssum = ssum; c.Wc = P[2 + 12 * L]; c.bc = P[3 + 12 * L]; c.O = d.odim; c.act = d.act;
    c.ds = ds_ws; c.dW_part = part[2 + 6 * L]; c.db_part = part[3 + 6 * L]; c.M = M;
    mdtc_train_cls_bwd_kernel<C><<<S, NT, 0, st>>>(c);
    if ((rc = check_launch("mdtc_train_cls_bwd_kernel"))) return rc;
  }
  for (int b = L - 1; b >= 0; --b) {
    GStatArgs g{};
    g.dy = dy(b); g.y = y(b); g.a = a2(b); g.stats = bstats(b, 2); g.part = gpart[0]; g.M = M;
    mdtc_train_gstat_kernel<C><<<S, NT, 0, st>>>(g);
    if ((rc = check_launch("mdtc_train_gstat_kernel"))) return rc;
    const int q = 2 + 6 * b;                                  // this block's first sliced gradient
    for (int which = 1; which >= 0; --which) {                // conv2 (BN2 -> dh1), then pointwise (BN1 -> dn0)
      PwBwdArgs p{};
      p.up = which == 1 ? dy(b) : t1;
      p.ymask = which == 1 ? y(b) : nullptr;
      p.bo = bng(b, which + 1, which == 1 ? a2(b) : a1(b), gpart[which == 1 ? 0 : 1]);
      p.W = P[pidx(b, which == 1 ? 8 : 4)];
      p.a_in = which == 1 ? a1(b) : a0(b);
      p.st_in = bstats(b, which);
      p.gamma_in = P[pidx(b, which == 1 ? 6 : 2)];
      p.beta_in = P[pidx(b, which == 1 ? 7 : 3)];
      p.relu_in = which;
      p.dW_part = part[q + (which == 1 ? 4 : 2)];
      p.db_part = part[q + (which == 1 ? 5 : 3)];
      p.dn = which == 1 ? t1 : t2;
      p.part = gpart[which == 1 ? 1 : 0];
      p.M = M;
      mdtc_train_pw_bwd_kernel<C><<<S, NT, 0, st>>>(p);
      if ((rc = check_launch("mdtc_train_pw_bwd_kernel"))) return rc;
    }
    DwBwdArgs a{};
    a.dn0 = t2; a.b0 = bng(b, 0, a0(b), gpart[0]);
    a.w = P[pidx(b, 0)]; a.in = y(b - 1);
    a.dy = dy(b); a.y = y(b);
    a.ds = b > 0 && mdtc_stack_end(b - 1, d.stack_size) ? ds : nullptr;
    a.mask_in = b == 0;
    a.d_in = dyr[b > 0 ? (b - 1) % 2 : 1];                   // dy(b - 1): block b - 1 < L - 1 is no last block
    a.dw_part = part[q]; a.db_part = part[q + 1];
    a.M = M; a.T = T; a.K = d.K; a.dil = d.dil[b];
    mdtc_train_dw_bwd_kernel<C><<<S, NT, 0, st>>>(a);
    if ((rc = check_launch("mdtc_train_dw_bwd_kernel"))) return rc;
  }
  {
    PreBwdArgs p{};
    p.d = dyr[1]; p.x = feats; p.mean = cmvn_mean; p.istd = cmvn_istd; p.norm_var = d.norm_var;
    p.dW_part = part[0]; p.db_part = part[1]; p.M = M; p.idim = d.idim;
    mdtc_train_pre_bwd_kernel<C><<<S, NT, 0, st>>>(p);
    if ((rc = check_launch("mdtc_train_pre_bwd_kernel"))) return rc;
  }
  ReduceArgs r{};
  int nj = 0;
  long long most = 0;
  auto job = [&](int pi, int gi) {
    r.j[nj].part = part[pi]; r.j[nj].out = grads[gi]; r.j[nj].n = (int)sizes[pi];
    most = std::max(most, sizes[pi]);
    ++nj;
  };
  job(0, 0); job(1, 1);
  for (int b = 0; b < L; ++b) {
    const int q = 2 + 6 * b;
    job(q, pidx(b, 0)); job(q + 1, pidx(b, 1)); job(q + 2, pidx(b, 4)); job(q + 3, pidx(b, 5));
    job(q + 4, pidx(b, 8)); job(q + 5, pidx(b, 9));
  }
  if (d.odim > 0) { job(2 + 6 * L, 2 + 12 * L); job(3 + 6 * L, 3 + 12 * L); }
  const int bx = (int)std::min<long long>((most + 255) / 256, 32);
  mdtc_train_reduce_kernel<<<dim3(bx, nj), 256, 0, st>>>(r);
  return check_launch("mdtc_train_reduce_kernel");
}

}  // namespace

long long mdtc_train_saved_floats(const MdtcTrainDims& d, long long M) {
  return 12LL * d.L * d.C + M * d.C * (4LL * d.L + 2);
}

float* mdtc_train_stack_sum(const MdtcTrainDims& d, long long M, float* saved, void* workspace) {
  const long long MC = M * d.C;
  if (saved) return saved + 12LL * d.L * d.C + MC * (1 + 4LL * d.L);
  return (float*)((double*)workspace + 3LL * S * 2 * d.C) + 5 * MC;
}

long long mdtc_train_workspace_bytes(const MdtcTrainDims& d, long long M, bool save) {
  return 48LL * S * d.C + (save ? 0 : 24LL * M * d.C);
}

long long mdtc_backward_workspace_bytes(const MdtcTrainDims& d, long long M) {
  return 32LL * S * d.C + 4 * 5 * M * d.C + 8LL * S * sliced_total(d);
}

int mdtc_train_forward_launch(const MdtcTrainDims& d, const float* feats, const float* const* params,
                              const float* cmvn_mean, const float* cmvn_istd, float* const* running, const double* bn,
                              float* out, float* out_cache, float* saved, void* workspace, int B, int T,
                              cudaStream_t st) {
  if (d.C == 64)
    return forward_t<64>(d, feats, params, cmvn_mean, cmvn_istd, running, bn, out, out_cache, saved, workspace, B, T, st);
  return forward_t<32>(d, feats, params, cmvn_mean, cmvn_istd, running, bn, out, out_cache, saved, workspace, B, T, st);
}

int mdtc_backward_launch(const MdtcTrainDims& d, const float* feats, const float* const* params,
                         const float* cmvn_mean, const float* cmvn_istd, const float* saved, const float* grad_out,
                         int B, int T, float* const* grads, void* workspace, cudaStream_t st) {
  if (d.C == 64)
    return backward_t<64>(d, feats, params, cmvn_mean, cmvn_istd, saved, grad_out, B, T, grads, workspace, st);
  return backward_t<32>(d, feats, params, cmvn_mean, cmvn_istd, saved, grad_out, B, T, grads, workspace, st);
}

}  // namespace wekws
