// TCN / DS-TCN training (wekws/utils/executor.py Executor.train through wekws/model/tcn.py): the training-mode
// forward, with every BatchNorm normalising by the statistics of the batch and updating its running statistics and
// every block's Dropout applying a mask that is a pure function of a seed (tcn_train.h dropout_keep), and the backward
// to every parameter of the reference's TCN / DS-TCN model with the per-frame linear classifier.
//
// FP32 FMA throughout.  Activations are channel-last (M = B * T rows of C floats), every frame a row, padding
// included, as torch's BatchNorm1d takes them.  Batch statistics follow train_common.cuh: the row-sliced launches run
// TRAIN_SLICES CTAs, each forming its slice's sums in double.  Weight gradients are tiles of dW = G^T X over fixed
// row ranges, accumulated in FP32 over 256 rows and in double across them; the ranges' double partials and the
// per-slice partials of the vector gradients are added in order by one final launch.  No atomics: equal inputs give
// equal bits.
//
// Block l (input x; x_0 the preprocessing output, x_{l+1} = y_l), dilation 2^l, causal zero left padding:
//   dense: a = conv(x) + b;                     y = x + D_l(relu(BN(a)))
//   ds:    a0 = dwconv(x) + b0, z0 = relu(BN0(a0)), a1 = W1 z0 + b1;   y = x + D_l(relu(BN1(a1)))
// y is formed on load by the next consumer (the next block's conv, or the classifier), which also stores it once.
// The saved buffer keeps the pre-BatchNorm tensors, the block outputs and the preprocessing output; x_hat and the
// Dropout masks are recomputed in the backward.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "tcn_train.h"
#include "train_common.cuh"

namespace wekws {

namespace {

using namespace train;
constexpr int S = TRAIN_SLICES;
constexpr int NT = TRAIN_NT;
constexpr int RT = 64, KC = 16;         // full-width GEMM: 64-row tiles, 16-deep reduction chunks
constexpr int WG_ROWS = 256;            // weight-gradient GEMM: FP32 accumulation length before the double add

// per-channel constants a kernel folds in its prologue
template <int C>
struct Fold {
  float sc[C], sh[C], sb[C];            // the forward affine of the BatchNorm whose output is formed on load
  float sc2[C], sh2[C], sb2[C];         // a second one (backward: the BatchNorm in front of the GEMM's input)
  double k1[C], mg[C], mgx[C], mean[C], inv[C];   // the gradient fold of the BatchNorm behind the GEMM's output
  double mean2[C], inv2[C];
  double tmp[2 * C];
};

template <int C>
struct FwSmem {
  union {
    struct {
      float As[KC][RT];
      float Ws[KC][C];
    } g;
    double red[16][C];
  } u;
  Fold<C> f;
};

// the affine of a BatchNorm from stored (mean, invstd): the forward's bits
template <int C>
__device__ inline void affine_from_stats(const double* st, const float* gamma, const float* beta, float* sc, float* sh,
                                         float* sb, double* mean, double* inv) {
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    bn_affine(st[c], st[C + c], gamma[c], sc[c], sh[c]);
    sb[c] = beta[c];
    if (mean != nullptr) {
      mean[c] = st[c];
      inv[c] = st[C + c];
    }
  }
}

// A block's output recomputed from its pre-BatchNorm tensor: y = res + D(relu(BN(a)))
struct BlockOut {
  const float* a; const float* res;      // a == nullptr: y = res (the preprocessing output)
  uint64_t seed; uint32_t theta; float scale; int layer;
};

__device__ inline float block_out(const BlockOut& o, const float* sc, const float* sh, const float* sb, long long r,
                                  int c, int C, int T) {
  const long long i = r * C + c;
  if (o.a == nullptr) return o.res[i];
  const int b = (int)(r / T), t = (int)(r % T);
  const float n = fmaxf(bn_apply(o.a[i], sh[c], sc[c], sb[c]), 0.f);
  const float y = dropout_keep(o.seed, o.layer, b, t, c, o.theta) ? n * o.scale : 0.f;
  return y + o.res[i];
}

// The gradient into a block's last pre-BatchNorm tensor a from the gradient gy into its output:
// gn = gy * scale where kept and relu(BN(a)) > 0, else 0; ga = BN backward (gradient statistics folded in k1 / mg / mgx)
struct BlockGrad {
  const float* gy; const float* a;
  uint64_t seed; uint32_t theta; float scale; int layer;
};

__device__ inline float block_gn(const BlockGrad& g, const float* sc, const float* sh, const float* sb, long long r,
                                 int c, int C, int T) {
  const long long i = r * C + c;
  const int b = (int)(r / T), t = (int)(r % T);
  if (!(bn_apply(g.a[i], sh[c], sc[c], sb[c]) > 0.f) || !dropout_keep(g.seed, g.layer, b, t, c, g.theta)) return 0.f;
  return g.gy[i] * g.scale;
}

template <int C>
__device__ inline float block_ga(const BlockGrad& g, const Fold<C>& f, long long r, int c, int T) {
  const float gn = block_gn(g, f.sc, f.sh, f.sb, r, c, C, T);
  return (float)bn_grad<C>(gn, g.a[r * C + c], c, f.k1, f.mg, f.mgx, f.mean, f.inv);
}

// ---------------------------------------------------------------------------------------------------- GEMM cores
// out[r][n] = sum_q A(r, q) W(n, q) + bias(n) for the rows of this CTA's slice and all C columns; every A element is
// formed once.  Op: K, M, prologue(Fold&), a(Fold&, r, q), w(n, q), bias(n), epi(Fold&, r, n, v, d1, d2) -> stats
// when op.part != nullptr.
template <int C, class Op>
__global__ void __launch_bounds__(NT) tcn_train_fw_kernel(const Op op) {
  constexpr int CPT = C / 16;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FwSmem<C>& s = *reinterpret_cast<FwSmem<C>*>(smem_raw);
  op.prologue(s.f);
  __syncthreads();
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  float bias[CPT];
#pragma unroll
  for (int v = 0; v < CPT; ++v) bias[v] = op.bias(tx + 16 * v);
  double s1[CPT], s2[CPT];
#pragma unroll
  for (int v = 0; v < CPT; ++v) s1[v] = s2[v] = 0.0;
  const Rows sl = slice_rows(op.M);
  for (long long q0 = sl.r0; q0 < sl.r1; q0 += RT) {
    const int nr = (int)min((long long)RT, sl.r1 - q0);
    float acc[4][CPT];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < CPT; ++v) acc[u][v] = 0.f;
    for (int k0 = 0; k0 < op.K; k0 += KC) {
      __syncthreads();
      for (int e = tid; e < RT * KC; e += NT) {
        const int r = e / KC, kk = e % KC;
        s.u.g.As[kk][r] = r < nr && k0 + kk < op.K ? op.a(s.f, q0 + r, k0 + kk) : 0.f;
      }
      for (int e = tid; e < C * KC; e += NT) {
        const int n = e / KC, kk = e % KC;
        s.u.g.Ws[kk][n] = k0 + kk < op.K ? op.w(n, k0 + kk) : 0.f;
      }
      __syncthreads();
#pragma unroll 4
      for (int kk = 0; kk < KC; ++kk) {
        const float4 a4 = *reinterpret_cast<const float4*>(&s.u.g.As[kk][ty * 4]);
        const float av[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
        for (int v = 0; v < CPT; ++v) {
          const float wv = s.u.g.Ws[kk][tx + 16 * v];
#pragma unroll
          for (int u = 0; u < 4; ++u) acc[u][v] = fmaf(av[u], wv, acc[u][v]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int r = ty * 4 + u;
      if (r >= nr) continue;
#pragma unroll
      for (int v = 0; v < CPT; ++v) {
        double d1 = 0.0, d2 = 0.0;
        op.epi(s.f, q0 + r, tx + 16 * v, acc[u][v] + bias[v], d1, d2);
        s1[v] += d1;
        s2[v] += d2;
      }
    }
  }
  if (op.part == nullptr) return;
  // the 16 row groups' sums in group order
  for (int which = 0; which < 2; ++which) {
    __syncthreads();
#pragma unroll
    for (int v = 0; v < CPT; ++v) s.u.red[ty][tx + 16 * v] = which ? s2[v] : s1[v];
    __syncthreads();
    for (int c = tid; c < C; c += NT) {
      double t = 0.0;
      for (int q = 0; q < 16; ++q) t += s.u.red[q][c];
      op.part[(long long)blockIdx.x * 2 * C + which * C + c] = t;
    }
  }
}

// Weight gradient: part[z][n][q] = sum over the rows of range z of G(r, n) X(r, q), q < Q, plus the column q = Q of
// X = 1 (the bias) when op.bias.  Op: M, N, Q, bias, part, prologue(Fold&), g(Fold&, r, n), x(Fold&, r, q).
template <int C, class Op>
__global__ void __launch_bounds__(NT) tcn_train_wg_kernel(const Op op) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fold<C>& f = *reinterpret_cast<Fold<C>*>(smem_raw);
  __shared__ float Gs[16][64], Xs[16][64];
  op.prologue(f);
  __syncthreads();
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  const int n0 = blockIdx.x * 64, p0 = blockIdx.y * 64, Qp = op.Q + (op.bias ? 1 : 0);
  const long long rs = (op.M + gridDim.z - 1) / gridDim.z;
  const long long r0 = min(op.M, (long long)blockIdx.z * rs), r1 = min(op.M, r0 + rs);
  float acc[4][4];
  double accd[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f, accd[i][j] = 0.0;
  int since = 0;
  for (long long q0 = r0; q0 < r1; q0 += 16) {
    const int nr = (int)min(16LL, r1 - q0);
    __syncthreads();
    for (int e = tid; e < 16 * 64; e += NT) {
      const int r = e / 64, j = e % 64;
      const bool ok = r < nr;
      Gs[r][j] = ok && n0 + j < op.N ? op.g(f, q0 + r, n0 + j) : 0.f;
      const int q = p0 + j;
      Xs[r][j] = !ok || q >= Qp ? 0.f : q == op.Q ? 1.f : op.x(f, q0 + r, q);
    }
    __syncthreads();
#pragma unroll 4
    for (int r = 0; r < 16; ++r) {
      float gv[4], xv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) gv[i] = Gs[r][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) xv[j] = Xs[r][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(gv[i], xv[j], acc[i][j]);
    }
    since += 16;
    if (since == WG_ROWS) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) accd[i][j] += (double)acc[i][j], acc[i][j] = 0.f;
      since = 0;
    }
  }
  double* out = op.part + (long long)blockIdx.z * op.N * Qp;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + ty + 16 * i, q = p0 + tx + 16 * j;
      if (n < op.N && q < Qp) out[(long long)n * Qp + q] = accd[i][j] + (double)acc[i][j];
    }
}

// ---------------------------------------------------------------------------------------------------- forward ops
struct NoFold {
  template <class F> __device__ void prologue(F&) const {}
};

// preprocessing Linear(idim, C) + ReLU of the CMVN-normalised features
struct PreOp : NoFold {
  const float* x; const float* mean; const float* istd; int norm_var;
  const float* W; const float* b; float* h0;
  long long M; int K, C;
  double* part;
  template <class F> __device__ float a(const F&, long long r, int q) const {
    float v = x[r * K + q];
    if (mean != nullptr) {                       // wekws/model/cmvn.py: x - mean, then * istd if norm_var
      v = v - mean[q];
      if (norm_var) v = v * istd[q];
    }
    return v;
  }
  __device__ float w(int n, int q) const { return W[n * K + q]; }
  __device__ float bias(int n) const { return b[n]; }
  template <class F> __device__ void epi(F&, long long r, int n, float v, double&, double&) const {
    h0[r * C + n] = fmaxf(v, 0.f);
  }
};

// the previous block's BatchNorm folded from its slice sums (l > 0)
template <int C>
__device__ inline void fold_prev(const BnFold& f, bool on, long long M, Fold<C>& s) {
  if (on) fold_bn<C>(f, M, s.sc, s.sh, s.sb, s.tmp);
}

// The block input x_l formed on load; its row frame t of utterance b also goes to y_out (when kept) and to block l's
// out_cache columns (the last `pad` frames of [zeros(pad) | x_l]).
struct InputStore {
  float* y_out; float* cache; int cache_off, pad, ptot;
};

__device__ inline void store_input(const InputStore& s, long long r, int c, float v, int C, int T) {
  if (s.y_out != nullptr) s.y_out[r * C + c] = v;
  const int t = (int)(r % T);
  float* cache = s.cache + ((r / T) * C + c) * s.ptot + s.cache_off;
  const int j = s.pad - T + t;
  if (j >= 0) cache[j] = v;
  if (t == T - 1)
    for (int z = 0; z < s.pad - T; ++z) cache[z] = 0.f;
}

// dense block: a = conv_{K, d}(x_l) + b, x_l formed on load; a's slice stats
template <int C>
struct ConvOp {
  BlockOut in; BnFold fin; int fold_in;
  InputStore st;
  const float* W; const float* bconv; float* out;
  long long M; int K, T, taps, dil;
  double* part;
  __device__ void prologue(Fold<C>& f) const { fold_prev<C>(fin, fold_in, M, f); }
  __device__ float a(const Fold<C>& f, long long r, int q) const {
    const int j = q / C, c = q % C, t = (int)(r % T), sh = (taps - 1 - j) * dil;
    if (t - sh < 0) return 0.f;
    const float v = block_out(in, f.sc, f.sh, f.sb, r - sh, c, C, T);
    if (sh == 0) store_input(st, r, c, v, C, T);
    return v;
  }
  __device__ float w(int n, int q) const { return W[(n * C + q % C) * taps + q / C]; }
  __device__ float bias(int n) const { return bconv[n]; }
  __device__ void epi(Fold<C>&, long long r, int n, float v, double& d1, double& d2) const {
    out[r * C + n] = v;
    d1 = (double)v;
    d2 = (double)v * (double)v;
  }
};

// ds block: a1 = W1 relu(BN0(a0)) + b1; a1's slice stats
template <int C>
struct PwOp {
  const float* a0; BnFold f0;
  const float* W; const float* b1; float* out;
  long long M; int K;
  double* part;
  __device__ void prologue(Fold<C>& f) const { fold_bn<C>(f0, M, f.sc, f.sh, f.sb, f.tmp); }
  __device__ float a(const Fold<C>& f, long long r, int q) const {
    return fmaxf(bn_apply(a0[r * C + q], f.sh[q], f.sc[q], f.sb[q]), 0.f);
  }
  __device__ float w(int n, int q) const { return W[n * C + q]; }
  __device__ float bias(int n) const { return b1[n]; }
  __device__ void epi(Fold<C>&, long long r, int n, float v, double& d1, double& d2) const {
    out[r * C + n] = v;
    d1 = (double)v;
    d2 = (double)v * (double)v;
  }
};

// ds block: a0 = dwconv_{K, d}(x_l) + b0 with x_l formed on load (stored once, and its out_cache slice); a0's stats
struct DwArgs {
  BlockOut in; BnFold fin; int fold_in;
  InputStore st;
  const float* w; const float* bias; float* a0; double* part;
  long long M; int T, K, dil;
};

template <int C>
__global__ void __launch_bounds__(NT) tcn_train_dw_kernel(const DwArgs a) {
  constexpr int G = NT / C;
  __shared__ Fold<C> f;
  __shared__ double red[G][2][C];
  fold_prev<C>(a.fin, a.fold_in, a.M, f);
  const Rows sl = slice_rows(a.M);
  const int c = threadIdx.x % C, g = threadIdx.x / C;
  float w[TCN_TRAIN_MAX_K];
#pragma unroll
  for (int k = 0; k < TCN_TRAIN_MAX_K; ++k) w[k] = k < a.K ? a.w[c * a.K + k] : 0.f;
  const float bias = a.bias[c];
  double s1 = 0.0, sq = 0.0;
  for (long long r = sl.r0 + g; r < sl.r1; r += G) {
    const int t = (int)(r % a.T);
    float acc = bias, cur = 0.f;
#pragma unroll
    for (int k = 0; k < TCN_TRAIN_MAX_K; ++k) {
      if (k >= a.K) break;
      const int sh = (a.K - 1 - k) * a.dil;
      const float v = t - sh >= 0 ? block_out(a.in, f.sc, f.sh, f.sb, r - sh, c, C, a.T) : 0.f;
      acc = fmaf(w[k], v, acc);
      cur = v;                                      // the last tap is frame t itself
    }
    a.a0[r * C + c] = acc;
    s1 += (double)acc;
    sq += (double)acc * (double)acc;
    store_input(a.st, r, c, cur, C, a.T);
  }
  write_slice_stats<C, G>(red, g, c, s1, sq, a.part);
}

// classifier: out = act(Wc y + bc), y = the last block's output formed on load (and stored once)
struct ClsArgs {
  BlockOut in; BnFold fin;
  float* y_out;
  const float* Wc; const float* bc; float* out; int O, act;
  long long M; int T;
};

template <int C>
struct ClsSmem {
  float A[32][C + 1];
  float Ws[32][65];
  Fold<C> f;
};

template <int C>
__global__ void __launch_bounds__(NT) tcn_train_cls_kernel(const ClsArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ClsSmem<C>& s = *reinterpret_cast<ClsSmem<C>*>(smem_raw);
  fold_bn<C>(a.fin, a.M, s.f.sc, s.f.sh, s.f.sb, s.f.tmp);
  const Rows sl = slice_rows(a.M);
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  for (long long q0 = sl.r0; q0 < sl.r1; q0 += 32) {
    const int nr = (int)min(32LL, sl.r1 - q0);
    __syncthreads();
    for (int e = tid; e < 32 * C; e += NT) {
      const int r = e / C, c = e % C;
      float v = 0.f;
      if (r < nr) {
        v = block_out(a.in, s.f.sc, s.f.sh, s.f.sb, q0 + r, c, C, a.T);
        if (a.y_out != nullptr) a.y_out[(q0 + r) * C + c] = v;
      }
      s.A[r][c] = v;
    }
    for (int o0 = 0; o0 < a.O; o0 += 64) {
      float acc[2][4];
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = 0.f;
      for (int k0 = 0; k0 < C; k0 += 32) {
        __syncthreads();
        for (int e = tid; e < 32 * 64; e += NT) {
          const int o = e / 32, kk = e % 32;
          s.Ws[kk][o] = o0 + o < a.O ? a.Wc[(long long)(o0 + o) * C + k0 + kk] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < 32; ++kk) {
          const float x0 = s.A[ty * 2][k0 + kk], x1 = s.A[ty * 2 + 1][k0 + kk];
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            const float wv = s.Ws[kk][tx + 16 * v];
            acc[0][v] = fmaf(x0, wv, acc[0][v]);
            acc[1][v] = fmaf(x1, wv, acc[1][v]);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int r = ty * 2 + u;
        if (r >= nr) continue;
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const int o = o0 + tx + 16 * v;
          if (o >= a.O) continue;
          const float z = acc[u][v] + a.bc[o];
          a.out[(q0 + r) * a.O + o] = a.act ? 1.f / (1.f + expf(-z)) : z;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------- backward ops
// the gradient statistics of block l's last BatchNorm from gy = the gradient into its output, at element (r, c)
template <int C>
__device__ inline void gstat(const BlockGrad& g, const Fold<C>& f, long long r, int c, int T, float gy, double& d1,
                             double& d2) {
  const long long i = r * C + c;
  const int b = (int)(r / T), t = (int)(r % T);
  float gn = 0.f;
  if (bn_apply(g.a[i], f.sh2[c], f.sc2[c], f.sb2[c]) > 0.f && dropout_keep(g.seed, g.layer, b, t, c, g.theta))
    gn = gy * g.scale;
  d1 = (double)gn;
  d2 = (double)gn * (((double)g.a[i] - f.mean2[c]) * f.inv2[c]);
}

// classifier: gy_{L-1} = dz Wc, dz = g (1 - y) y for the sigmoid (torch's sigmoid_backward from the output y), with
// the gradient statistics of the last block's BatchNorm
template <int C>
struct ClsDxOp {
  const float* g; const float* y; int act;
  const float* Wc; float* gy;
  BlockGrad last; const double* st_last; const float* gamma_last; const float* beta_last;
  long long M; int K, T;
  double* part;
  __device__ void prologue(Fold<C>& f) const {
    affine_from_stats<C>(st_last, gamma_last, beta_last, f.sc2, f.sh2, f.sb2, f.mean2, f.inv2);
  }
  __device__ float a(const Fold<C>&, long long r, int o) const {
    const long long i = r * K + o;
    return act ? g[i] * (1.f - y[i]) * y[i] : g[i];
  }
  __device__ float w(int n, int o) const { return Wc[(long long)o * C + n]; }
  __device__ float bias(int) const { return 0.f; }
  __device__ void epi(Fold<C>& f, long long r, int n, float v, double& d1, double& d2) const {
    gy[r * C + n] = v;
    gstat<C>(last, f, r, n, T, v, d1, d2);
  }
};

// dWc, dbc: G = dz on load, X = y_{L-1}
template <int C>
struct WgCls {
  const float* g; const float* y; int act; const float* x;
  long long M; int N, Q, bias;
  double* part;
  __device__ void prologue(Fold<C>&) const {}
  __device__ float gfun(const Fold<C>&, long long r, int o) const {
    const long long i = r * N + o;
    return act ? g[i] * (1.f - y[i]) * y[i] : g[i];
  }
  __device__ float xfun(const Fold<C>&, long long r, int c) const { return x[r * C + c]; }
};

// ds block backward, pointwise: gz0 = ga1 W1, ga1 = BN1 backward of gn1 (stored for the weight gradient); then
// gn0 = gz0 [z0 > 0] with its statistics against BN0's x_hat
template <int C>
struct PwDxOp {
  BlockGrad gb; BnGrad bg1; const float* beta1;      // BN1: the block's last BatchNorm
  const double* st0; const float* gamma0; const float* beta0; const float* a0;
  const float* W1; float* ga1; float* gn0;
  long long M; int K, T;
  double* part;
  __device__ void prologue(Fold<C>& f) const {
    fold_bn_grad<C>(bg1, M, f.k1, f.mg, f.mgx, f.mean, f.inv, f.tmp);
    affine_from_stats<C>(bg1.stats, bg1.gamma, beta1, f.sc, f.sh, f.sb, nullptr, nullptr);
    affine_from_stats<C>(st0, gamma0, beta0, f.sc2, f.sh2, f.sb2, f.mean2, f.inv2);
  }
  __device__ float a(const Fold<C>& f, long long r, int o) const {
    const float v = block_ga<C>(gb, f, r, o, T);
    ga1[r * C + o] = v;
    return v;
  }
  __device__ float w(int n, int o) const { return W1[o * C + n]; }
  __device__ float bias(int) const { return 0.f; }
  __device__ void epi(Fold<C>& f, long long r, int n, float v, double& d1, double& d2) const {
    const long long i = r * C + n;
    const float g = bn_apply(a0[i], f.sh2[n], f.sc2[n], f.sb2[n]) > 0.f ? v : 0.f;   // torch's threshold_backward
    gn0[i] = g;
    d1 = (double)g;
    d2 = (double)g * (((double)a0[i] - f.mean2[n]) * f.inv2[n]);
  }
};

// dW1, db1: G = ga1, X = z0 = relu(BN0(a0))
template <int C>
struct WgPw {
  const float* ga1; const float* a0; const double* st0; const float* gamma0; const float* beta0;
  long long M; int N, Q, bias;
  double* part;
  __device__ void prologue(Fold<C>& f) const {
    affine_from_stats<C>(st0, gamma0, beta0, f.sc, f.sh, f.sb, nullptr, nullptr);
  }
  __device__ float gfun(const Fold<C>&, long long r, int n) const { return ga1[r * C + n]; }
  __device__ float xfun(const Fold<C>& f, long long r, int c) const {
    return fmaxf(bn_apply(a0[r * C + c], f.sh[c], f.sc[c], f.sb[c]), 0.f);
  }
};

// dense block backward: gx = gy + sum_j W_j^T ga[t + s_j] (ga = BN backward of gn, stored at shift 0 for the weight
// gradient); then either the preprocessing ReLU's mask (l == 0) or the previous block's gradient statistics
template <int C>
struct ConvDxOp {
  BlockGrad gb; BnGrad bg; const float* beta;
  const float* W; float* ga; float* gx; const float* h0; int first;
  BlockGrad prev; const double* st_prev; const float* gamma_prev; const float* beta_prev;
  long long M; int K, T, taps, dil;
  double* part;
  __device__ void prologue(Fold<C>& f) const {
    fold_bn_grad<C>(bg, M, f.k1, f.mg, f.mgx, f.mean, f.inv, f.tmp);
    affine_from_stats<C>(bg.stats, bg.gamma, beta, f.sc, f.sh, f.sb, nullptr, nullptr);
    if (!first) affine_from_stats<C>(st_prev, gamma_prev, beta_prev, f.sc2, f.sh2, f.sb2, f.mean2, f.inv2);
  }
  __device__ float a(const Fold<C>& f, long long r, int q) const {
    const int j = q / C, co = q % C, t = (int)(r % T), sh = (taps - 1 - j) * dil;
    if (t + sh >= T) return 0.f;
    const float v = block_ga<C>(gb, f, r + sh, co, T);
    if (sh == 0) ga[r * C + co] = v;
    return v;
  }
  __device__ float w(int n, int q) const { return W[((q % C) * C + n) * taps + q / C]; }
  __device__ float bias(int) const { return 0.f; }
  __device__ void epi(Fold<C>& f, long long r, int n, float v, double& d1, double& d2) const {
    const long long i = r * C + n;
    const float g = v + gb.gy[i];                   // the residual
    if (first) {
      gx[i] = h0[i] > 0.f ? g : 0.f;                // the preprocessing ReLU
      return;
    }
    gx[i] = g;
    gstat<C>(prev, f, r, n, T, g, d1, d2);
  }
};

// dense dW, db: G = ga, X(r, (j, ci)) = x_l(r - s_j, ci)
template <int C>
struct WgConv {
  const float* ga; const float* x;
  long long M; int N, Q, bias, T, taps, dil;
  double* part;
  __device__ void prologue(Fold<C>&) const {}
  __device__ float gfun(const Fold<C>&, long long r, int n) const { return ga[r * C + n]; }
  __device__ float xfun(const Fold<C>&, long long r, int q) const {
    const int j = q / C, c = q % C, t = (int)(r % T), sh = (taps - 1 - j) * dil;
    return t - sh >= 0 ? x[(r - sh) * C + c] : 0.f;
  }
};

// preprocessing dW, db: G = the masked gradient of h0, X = CMVN(x)
template <int C>
struct WgPre {
  const float* gh; const float* x; const float* mean; const float* istd; int norm_var;
  long long M; int N, Q, bias;
  double* part;
  __device__ void prologue(Fold<C>&) const {}
  __device__ float gfun(const Fold<C>&, long long r, int n) const { return gh[r * C + n]; }
  __device__ float xfun(const Fold<C>&, long long r, int q) const {
    float v = x[r * Q + q];
    if (mean != nullptr) {
      v = v - mean[q];
      if (norm_var) v = v * istd[q];
    }
    return v;
  }
};

// adapts the G / X ops to the wg kernel's interface
template <int C, class W>
struct Wg {
  W op;
  long long M; int N, Q, bias;
  double* part;
  __device__ void prologue(Fold<C>& f) const { op.prologue(f); }
  __device__ float g(const Fold<C>& f, long long r, int n) const { return op.gfun(f, r, n); }
  __device__ float x(const Fold<C>& f, long long r, int q) const { return op.xfun(f, r, q); }
};

// ds block backward, depthwise: ga0 = BN0 backward of gn0; gx = gy + sum_k w_k ga0[t + s_k] (within each utterance);
// tap and bias gradients as slice partials [C][K], [C]; then the preprocessing ReLU's mask (l == 0) or the previous
// block's gradient statistics
struct DwBwdArgs {
  const float* gn0; BnGrad b0;
  const float* w; const float* in; const float* gy; float* gx; int first;
  BlockGrad prev; const double* st_prev; const float* gamma_prev; const float* beta_prev; double* part;
  double* dw_part; double* db_part;
  long long M; int T, K, dil;
};

template <int C>
__global__ void __launch_bounds__(NT) tcn_train_dw_bwd_kernel(const DwBwdArgs a) {
  constexpr int G = NT / C, KP = TCN_TRAIN_MAX_K + 1;
  __shared__ Fold<C> f;
  __shared__ double red[G][KP][C];
  fold_bn_grad<C>(a.b0, a.M, f.k1, f.mg, f.mgx, f.mean, f.inv, f.tmp);
  if (!a.first) affine_from_stats<C>(a.st_prev, a.gamma_prev, a.beta_prev, f.sc2, f.sh2, f.sb2, f.mean2, f.inv2);
  __syncthreads();
  const int c = threadIdx.x % C, g = threadIdx.x / C;
  float w[TCN_TRAIN_MAX_K];
  double acc[KP];
#pragma unroll
  for (int k = 0; k < TCN_TRAIN_MAX_K; ++k) w[k] = k < a.K ? a.w[c * a.K + k] : 0.f;
#pragma unroll
  for (int k = 0; k < KP; ++k) acc[k] = 0.0;
  double s1 = 0.0, s2 = 0.0;
  auto da = [&](long long row) {
    const long long i = row * C + c;
    return bn_grad<C>(a.gn0[i], a.b0.a[i], c, f.k1, f.mg, f.mgx, f.mean, f.inv);
  };
  const Rows sl = slice_rows(a.M);
  for (long long r = sl.r0 + g; r < sl.r1; r += G) {
    const int t = (int)(r % a.T);
    const long long base = r - t, i = r * C + c;
    const double dself = da(r);
    float d = 0.f;
#pragma unroll
    for (int k = 0; k < TCN_TRAIN_MAX_K; ++k) {
      if (k >= a.K) break;
      const int sh = (a.K - 1 - k) * a.dil;
      if (t + sh < a.T) d = fmaf(w[k], (float)(sh == 0 ? dself : da(base + t + sh)), d);   // output t + sh read x[t]
      if (t - sh >= 0) acc[k] = fma(dself, (double)a.in[(base + t - sh) * C + c], acc[k]);
    }
    acc[TCN_TRAIN_MAX_K] += dself;
    d += a.gy[i];                                    // the residual
    if (a.first) {
      a.gx[i] = a.in[i] > 0.f ? d : 0.f;             // the preprocessing ReLU
    } else {
      a.gx[i] = d;
      double d1, d2;
      gstat<C>(a.prev, f, r, c, a.T, d, d1, d2);
      s1 += d1;
      s2 += d2;
    }
  }
  if (!a.first) {
    __shared__ double rs[G][2][C];
    write_slice_stats<C, G>(rs, g, c, s1, s2, a.part);
  }
#pragma unroll
  for (int k = 0; k < KP; ++k) red[g][k][c] = acc[k];
  __syncthreads();
  for (int e = threadIdx.x; e < (a.K + 1) * C; e += NT) {
    const int k = e / C, cc = e % C, kk = k < a.K ? k : TCN_TRAIN_MAX_K;
    double s = 0.0;
    for (int q = 0; q < G; ++q) s += red[q][kk][cc];
    if (k < a.K) a.dw_part[(long long)blockIdx.x * C * a.K + cc * a.K + k] = s;
    else a.db_part[(long long)blockIdx.x * C + cc] = s;
  }
}

// every weight / bias gradient: its partials added in order.  Job: part [Z][N][Qp]; out_w[n][q] at n * Q * taps-order,
// out_b[n] from q == Q when Qp > Q.
constexpr int MAX_JOBS = 4 + 4 * TCN_TRAIN_MAX_LAYERS;
struct ReduceJob {
  const double* part;
  float* w; float* b;
  int N, Q, Qp, Z, taps, C;             // taps > 1: q = j * C + ci -> w[(n * C + ci) * taps + j]
};
struct ReduceArgs {
  ReduceJob j[MAX_JOBS];
};

__global__ void tcn_train_reduce_kernel(const ReduceArgs a) {
  const ReduceJob& jb = a.j[blockIdx.y];
  const long long n = (long long)jb.N * jb.Qp;
  for (long long e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int z = 0; z < jb.Z; ++z) s += jb.part[z * n + e];
    const int o = (int)(e / jb.Qp), q = (int)(e % jb.Qp);
    if (q == jb.Q) jb.b[o] = (float)s;
    else if (jb.taps > 1) jb.w[((long long)o * jb.C + q % jb.C) * jb.taps + q / jb.C] = (float)s;
    else jb.w[(long long)o * jb.Q + q] = (float)s;
  }
}

__global__ void dropout_mask_kernel(uint64_t seed, long long n, int T, int C, int layer, uint32_t theta, uint8_t* out) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / C;
    out[e] = dropout_keep(seed, layer, (int)(r / T), (int)(r % T), (int)(e % C), theta) ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------------------------- host side
inline int pidx(const TcnTrainDims& d, int l, int k) { return 2 + tcn_train_params_per_block(d.ds) * l + k; }
inline int dil(int l) { return 1 << l; }

// The weight-gradient GEMMs' row ranges: enough CTAs for the device, fixed by the shape alone
int wg_splits(int N, int Qp, long long M) {
  const long long tiles = (long long)((N + 63) / 64) * ((Qp + 63) / 64);
  long long z = (264 + tiles - 1) / tiles;
  z = std::min<long long>(z, std::max<long long>(1, M / WG_ROWS));
  return (int)std::max<long long>(1, std::min<long long>(z, 64));
}

// every reduce job's (N, Qp, taps) in order: per block [dense: conv W + b | ds: dw taps, dw bias (slice partials),
// pointwise W + b], then the preprocessing W + b and the classifier W + b
struct Job {
  int N, Q, Qp, Z, taps;
};
std::vector<Job> jobs(const TcnTrainDims& d, long long M) {
  std::vector<Job> v;
  const int C = d.C;
  auto wg = [&](int N, int Q, int taps) { v.push_back({N, Q, Q + 1, wg_splits(N, Q + 1, M), taps}); };
  for (int l = 0; l < d.L; ++l) {
    if (d.ds) {
      v.push_back({C, d.K, d.K, S, 1});        // taps [C][K] per slice
      v.push_back({C, 1, 1, S, 1});            // bias [C] per slice (as an N x 1 job whose column 0 is the weight)
      wg(C, C, 1);
    } else {
      wg(C, d.K * C, d.K);
    }
  }
  wg(C, d.idim, 1);
  wg(d.odim, C, 1);
  return v;
}

long long partial_doubles(const std::vector<Job>& js) {
  long long s = 0;
  for (const Job& j : js) s += (long long)j.Z * j.N * j.Qp;
  return s;
}

template <auto kernel, class Arg>
int launch_dyn(dim3 grid, size_t smem, const Arg& a, cudaStream_t st, const char* name) {
  if (const int rc = opt_in_smem((const void*)kernel, smem)) return rc;
  kernel<<<grid, NT, smem, st>>>(a);
  return check_launch(name);
}

template <int C, class W>
int launch_wg(const W& w, long long M, int N, int Q, int Z, double* part, cudaStream_t st) {
  Wg<C, W> g{w, M, N, Q, 1, part};
  const dim3 grid((N + 63) / 64, (Q + 1 + 63) / 64, Z);
  return launch_dyn<tcn_train_wg_kernel<C, Wg<C, W>>>(grid, sizeof(Fold<C>), g, st, "tcn_train_wg_kernel");
}

// the saved buffer: [each BatchNorm's (mean, invstd) x C doubles][h0][per block its pre-BatchNorm tensors (ds: a0, a1;
// dense: a) and its output y]
struct Layout {
  const TcnTrainDims& d; long long MC; float* base;
  int per() const { return d.ds ? 3 : 2; }
  double* stats(int l, int which) const { return (double*)base + (long long)((d.ds ? 2 : 1) * l + which) * 2 * d.C; }
  float* act() const { return base + 4LL * tcn_train_num_bns(d) * d.C; }
  float* h0() const { return act(); }
  float* pre(int l, int which) const { return act() + MC * (1 + (long long)per() * l + which); }
  float* y(int l) const { return l < 0 ? h0() : act() + MC * (1 + (long long)per() * l + per() - 1); }
};

template <int C>
int forward_t(const TcnTrainDims& d, const TcnDropout& drop, const float* feats, const float* const* P,
              const float* cmvn_mean, const float* cmvn_istd, float* const* running, const double* bn, float* out,
              float* out_cache, float* saved, void* workspace, int B, int T, cudaStream_t st) {
  const long long M = (long long)B * T, MC = M * C;
  const int L = d.L, nbn = d.ds ? 2 : 1;
  double* part[2] = {(double*)workspace, (double*)workspace + 2LL * S * C};
  float* ws = (float*)((double*)workspace + 4LL * S * C);
  const Layout lay{d, MC, saved};
  // without `saved`: rings in the workspace (the block outputs in two slots, h0 in slot 0; pre-BN tensors in two)
  auto y = [&](int l) { return saved ? lay.y(l) : ws + MC * ((l + 1) % 2); };
  auto pre = [&](int l, int which) {
    return saved ? lay.pre(l, which) : ws + MC * (2 + (d.ds ? which : l % 2));
  };
  auto fold = [&](int l, int which, const double* p) {
    const int k = nbn * l + which;
    BnFold f{};
    f.part = p;
    f.gamma = P[pidx(d, l, which == 0 ? 2 : 6)];
    f.beta = P[pidx(d, l, which == 0 ? 3 : 7)];
    f.run_mean = running[2 * k];
    f.run_var = running[2 * k + 1];
    f.momentum = bn[2 * k];
    f.eps = bn[2 * k + 1];
    f.stats = saved ? lay.stats(l, which) : nullptr;
    return f;
  };
  auto last_part = [&](int l) { return d.ds ? part[1] : part[l % 2]; };    // the slice sums of block l's last BN
  auto block_out_of = [&](int l) {                  // y_l as the next consumer forms it
    BlockOut o{};
    o.a = pre(l, nbn - 1); o.res = y(l - 1);
    o.seed = drop.seed; o.theta = drop.theta[l]; o.scale = drop.scale[l]; o.layer = l;
    return o;
  };
  auto input_of = [&](int l) {                      // x_l: y_{l-1}, or h0
    if (l > 0) return block_out_of(l - 1);
    BlockOut o{};
    o.res = y(-1);
    return o;
  };
  const size_t fw = sizeof(FwSmem<C>);
  int rc;
  {
    PreOp p{};
    p.x = feats; p.mean = cmvn_mean; p.istd = cmvn_istd; p.norm_var = d.norm_var;
    p.W = P[0]; p.b = P[1]; p.h0 = y(-1); p.M = M; p.K = d.idim; p.C = C;
    if ((rc = launch_dyn<tcn_train_fw_kernel<C, PreOp>>(dim3(S), fw, p, st, "tcn_train_fw_kernel"))) return rc;
  }
  for (int l = 0; l < L; ++l) {
    InputStore is{};
    is.y_out = l > 0 ? y(l - 1) : nullptr;
    is.cache = out_cache; is.cache_off = (d.K - 1) * (dil(l) - 1); is.pad = (d.K - 1) * dil(l); is.ptot = d.pad_total;
    if (d.ds) {
      DwArgs a{};
      a.in = input_of(l);
      if (l > 0) { a.fin = fold(l - 1, 1, part[1]); a.fold_in = 1; }
      a.st = is;
      a.w = P[pidx(d, l, 0)]; a.bias = P[pidx(d, l, 1)]; a.a0 = pre(l, 0); a.part = part[0];
      a.M = M; a.T = T; a.K = d.K; a.dil = dil(l);
      tcn_train_dw_kernel<C><<<S, NT, 0, st>>>(a);
      if ((rc = check_launch("tcn_train_dw_kernel"))) return rc;
      PwOp<C> q{};
      q.a0 = pre(l, 0); q.f0 = fold(l, 0, part[0]);
      q.W = P[pidx(d, l, 4)]; q.b1 = P[pidx(d, l, 5)]; q.out = pre(l, 1); q.M = M; q.K = C; q.part = part[1];
      if ((rc = launch_dyn<tcn_train_fw_kernel<C, PwOp<C>>>(dim3(S), fw, q, st, "tcn_train_fw_kernel"))) return rc;
    } else {
      ConvOp<C> c{};
      c.in = input_of(l);
      if (l > 0) { c.fin = fold(l - 1, 0, last_part(l - 1)); c.fold_in = 1; }
      c.st = is;
      c.W = P[pidx(d, l, 0)]; c.bconv = P[pidx(d, l, 1)]; c.out = pre(l, 0);
      c.M = M; c.K = d.K * C; c.T = T; c.taps = d.K; c.dil = dil(l); c.part = last_part(l);
      if ((rc = launch_dyn<tcn_train_fw_kernel<C, ConvOp<C>>>(dim3(S), fw, c, st, "tcn_train_fw_kernel"))) return rc;
    }
  }
  ClsArgs c{};
  c.in = block_out_of(L - 1); c.fin = fold(L - 1, nbn - 1, last_part(L - 1));
  c.y_out = saved ? lay.y(L - 1) : nullptr;
  c.Wc = P[pidx(d, L, 0)]; c.bc = P[pidx(d, L, 1)]; c.out = out; c.O = d.odim; c.act = d.act; c.M = M; c.T = T;
  return launch_dyn<tcn_train_cls_kernel<C>>(dim3(S), sizeof(ClsSmem<C>), c, st, "tcn_train_cls_kernel");
}

template <int C>
int backward_t(const TcnTrainDims& d, const TcnDropout& drop, const float* feats, const float* const* P,
               const float* cmvn_mean, const float* cmvn_istd, const float* saved, const float* out,
               const float* grad_out, int B, int T, float* const* grads, void* workspace, cudaStream_t st) {
  const long long M = (long long)B * T, MC = M * C;
  const int L = d.L, nbn = d.ds ? 2 : 1;
  const Layout lay{d, MC, const_cast<float*>(saved)};
  // workspace: [gradient statistics x 2][gy x 2][ga][gn0][the partials of every reduce job, in order, as doubles]
  double* gpart[2] = {(double*)workspace, (double*)workspace + 2LL * S * C};
  float* gyb[2] = {(float*)((double*)workspace + 4LL * S * C), nullptr};
  gyb[1] = gyb[0] + MC;
  float* ga = gyb[0] + 2 * MC;
  float* gn0 = gyb[0] + 3 * MC;
  const std::vector<Job> js = jobs(d, M);
  std::vector<double*> jp(js.size());
  double* w = (double*)(gyb[0] + 4 * MC);
  for (size_t i = 0; i < js.size(); ++i) { jp[i] = w; w += (long long)js[i].Z * js[i].N * js[i].Qp; }
  auto gy = [&](int l) { return gyb[(L - 1 - l) % 2]; };                  // the gradient into y_l
  auto gamma = [&](int l, int which) { return P[pidx(d, l, which == 0 ? 2 : 6)]; };
  auto beta = [&](int l, int which) { return P[pidx(d, l, which == 0 ? 3 : 7)]; };
  auto bgrad = [&](int l) {                          // the gradient into block l's last pre-BN tensor, from gy(l)
    BlockGrad g{};
    g.gy = gy(l); g.a = lay.pre(l, nbn - 1);
    g.seed = drop.seed; g.theta = drop.theta[l]; g.scale = drop.scale[l]; g.layer = l;
    return g;
  };
  auto bng = [&](int l, int which, const float* a, const double* gp) {
    BnGrad g{};
    g.a = a; g.stats = lay.stats(l, which); g.gamma = gamma(l, which); g.gpart = gp;
    g.dgamma = grads[pidx(d, l, which == 0 ? 2 : 6)];
    g.dbeta = grads[pidx(d, l, which == 0 ? 3 : 7)];
    return g;
  };
  const size_t fw = sizeof(FwSmem<C>);
  int rc;
  {
    ClsDxOp<C> c{};
    c.g = grad_out; c.y = out; c.act = d.act; c.Wc = P[pidx(d, L, 0)]; c.gy = gy(L - 1);
    c.last = bgrad(L - 1); c.st_last = lay.stats(L - 1, nbn - 1);
    c.gamma_last = gamma(L - 1, nbn - 1); c.beta_last = beta(L - 1, nbn - 1);
    c.M = M; c.K = d.odim; c.T = T; c.part = gpart[0];
    if ((rc = launch_dyn<tcn_train_fw_kernel<C, ClsDxOp<C>>>(dim3(S), fw, c, st, "tcn_train_fw_kernel"))) return rc;
    const size_t j = js.size() - 1;
    WgCls<C> g{};
    g.g = grad_out; g.y = out; g.act = d.act; g.x = lay.y(L - 1); g.M = M; g.N = d.odim; g.Q = C;
    if ((rc = launch_wg<C>(g, M, d.odim, C, js[j].Z, jp[j], st))) return rc;
  }
  for (int l = L - 1; l >= 0; --l) {
    const bool first = l == 0;
    float* gx = first ? gyb[(L - l) % 2] : gy(l - 1);
    BlockGrad prev{};
    if (!first) prev = bgrad(l - 1);
    if (d.ds) {
      const int j0 = 3 * l;
      PwDxOp<C> p{};
      p.gb = bgrad(l); p.bg1 = bng(l, 1, lay.pre(l, 1), gpart[0]); p.beta1 = beta(l, 1);
      p.st0 = lay.stats(l, 0); p.gamma0 = gamma(l, 0); p.beta0 = beta(l, 0); p.a0 = lay.pre(l, 0);
      p.W1 = P[pidx(d, l, 4)]; p.ga1 = ga; p.gn0 = gn0; p.M = M; p.K = C; p.T = T; p.part = gpart[1];
      if ((rc = launch_dyn<tcn_train_fw_kernel<C, PwDxOp<C>>>(dim3(S), fw, p, st, "tcn_train_fw_kernel"))) return rc;
      WgPw<C> g{};
      g.ga1 = ga; g.a0 = lay.pre(l, 0); g.st0 = lay.stats(l, 0); g.gamma0 = gamma(l, 0); g.beta0 = beta(l, 0);
      if ((rc = launch_wg<C>(g, M, C, C, js[j0 + 2].Z, jp[j0 + 2], st))) return rc;
      DwBwdArgs a{};
      a.gn0 = gn0; a.b0 = bng(l, 0, lay.pre(l, 0), gpart[1]);
      a.w = P[pidx(d, l, 0)]; a.in = lay.y(l - 1); a.gy = gy(l); a.gx = gx; a.first = first;
      a.prev = prev;
      if (!first) { a.st_prev = lay.stats(l - 1, 1); a.gamma_prev = gamma(l - 1, 1); a.beta_prev = beta(l - 1, 1); }
      a.part = gpart[0]; a.dw_part = jp[j0]; a.db_part = jp[j0 + 1];
      a.M = M; a.T = T; a.K = d.K; a.dil = dil(l);
      tcn_train_dw_bwd_kernel<C><<<S, NT, 0, st>>>(a);
      if ((rc = check_launch("tcn_train_dw_bwd_kernel"))) return rc;
    } else {
      ConvDxOp<C> c{};
      c.gb = bgrad(l); c.bg = bng(l, 0, lay.pre(l, 0), gpart[(L - 1 - l) % 2]); c.beta = beta(l, 0);
      c.W = P[pidx(d, l, 0)]; c.ga = ga; c.gx = gx; c.h0 = lay.h0(); c.first = first;
      c.prev = prev;
      if (!first) { c.st_prev = lay.stats(l - 1, 0); c.gamma_prev = gamma(l - 1, 0); c.beta_prev = beta(l - 1, 0); }
      c.M = M; c.K = d.K * C; c.T = T; c.taps = d.K; c.dil = dil(l); c.part = gpart[(L - l) % 2];
      if ((rc = launch_dyn<tcn_train_fw_kernel<C, ConvDxOp<C>>>(dim3(S), fw, c, st, "tcn_train_fw_kernel"))) return rc;
      WgConv<C> g{};
      g.ga = ga; g.x = lay.y(l - 1); g.T = T; g.taps = d.K; g.dil = dil(l);
      if ((rc = launch_wg<C>(g, M, C, d.K * C, js[l].Z, jp[l], st))) return rc;
    }
  }
  {
    const size_t j = js.size() - 2;
    WgPre<C> g{};
    g.gh = gyb[L % 2]; g.x = feats; g.mean = cmvn_mean; g.istd = cmvn_istd; g.norm_var = d.norm_var; g.Q = d.idim;
    if ((rc = launch_wg<C>(g, M, C, d.idim, js[j].Z, jp[j], st))) return rc;
  }
  ReduceArgs r{};
  long long most = 0;
  const int nj = (int)js.size();
  for (int i = 0; i < nj; ++i) {
    ReduceJob& jb = r.j[i];
    jb.part = jp[i]; jb.N = js[i].N; jb.Q = js[i].Q; jb.Qp = js[i].Qp; jb.Z = js[i].Z; jb.taps = js[i].taps; jb.C = C;
    most = std::max(most, (long long)js[i].N * js[i].Qp);
  }
  for (int l = 0; l < L; ++l) {
    if (d.ds) {
      r.j[3 * l].w = grads[pidx(d, l, 0)];
      r.j[3 * l + 1].w = grads[pidx(d, l, 1)];
      r.j[3 * l + 2].w = grads[pidx(d, l, 4)]; r.j[3 * l + 2].b = grads[pidx(d, l, 5)];
    } else {
      r.j[l].w = grads[pidx(d, l, 0)]; r.j[l].b = grads[pidx(d, l, 1)];
    }
  }
  r.j[nj - 2].w = grads[0]; r.j[nj - 2].b = grads[1];
  r.j[nj - 1].w = grads[pidx(d, L, 0)]; r.j[nj - 1].b = grads[pidx(d, L, 1)];
  const int bx = (int)std::min<long long>((most + 255) / 256, 64);
  tcn_train_reduce_kernel<<<dim3(bx, nj), 256, 0, st>>>(r);
  return check_launch("tcn_train_reduce_kernel");
}

}  // namespace

long long tcn_train_saved_floats(const TcnTrainDims& d, long long M) {
  return 4LL * tcn_train_num_bns(d) * d.C + M * d.C * (1 + (long long)d.L * (d.ds ? 3 : 2));
}

long long tcn_train_workspace_bytes(const TcnTrainDims& d, long long M, bool save) {
  return 32LL * S * d.C + (save ? 0 : 16LL * M * d.C);
}

long long tcn_backward_workspace_bytes(const TcnTrainDims& d, long long M) {
  return 32LL * S * d.C + 16LL * M * d.C + 8LL * partial_doubles(jobs(d, M));
}

int tcn_train_forward_launch(const TcnTrainDims& d, const TcnDropout& drop, const float* feats,
                             const float* const* params, const float* cmvn_mean, const float* cmvn_istd,
                             float* const* running, const double* bn, float* out, float* out_cache, float* saved,
                             void* workspace, int B, int T, cudaStream_t st) {
  if (d.C == 64)
    return forward_t<64>(d, drop, feats, params, cmvn_mean, cmvn_istd, running, bn, out, out_cache, saved, workspace,
                         B, T, st);
  return forward_t<256>(d, drop, feats, params, cmvn_mean, cmvn_istd, running, bn, out, out_cache, saved, workspace,
                        B, T, st);
}

int tcn_backward_launch(const TcnTrainDims& d, const TcnDropout& drop, const float* feats, const float* const* params,
                        const float* cmvn_mean, const float* cmvn_istd, const float* saved, const float* out,
                        const float* grad_out, int B, int T, float* const* grads, void* workspace, cudaStream_t st) {
  if (d.C == 64)
    return backward_t<64>(d, drop, feats, params, cmvn_mean, cmvn_istd, saved, out, grad_out, B, T, grads, workspace,
                          st);
  return backward_t<256>(d, drop, feats, params, cmvn_mean, cmvn_istd, saved, out, grad_out, B, T, grads, workspace,
                         st);
}

int dropout_mask_launch(uint64_t seed, long long B, long long T, int C, int layer, uint32_t theta, uint8_t* out,
                        cudaStream_t st) {
  const long long n = B * T * C;
  if (n == 0) return 0;
  const int grid = (int)std::min<long long>((n + 255) / 256, 4096);
  dropout_mask_kernel<<<grid, 256, 0, st>>>(seed, n, (int)T, C, layer, theta, out);
  return check_launch("dropout_mask_kernel");
}

}  // namespace wekws
