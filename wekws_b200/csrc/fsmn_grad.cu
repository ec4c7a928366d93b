// FSMN training (wekws/utils/executor.py Executor.train through wekws/model/fsmn.py): the parameter pack from device
// tensors and the backward of the fused forward (fsmn.cu) to every parameter of the reference's FSMN.
//
// FP32 FMA throughout, as the forward (the widths 140 / 250 / 2599 of fsmn_ctc.yaml are not tensor-core shaped).
// Rows are the M = B * T frames, padding included, as torch's autograd takes them.  Every weight gradient
// dW = dY^T X (and db = column sums of dY) is split into FSMN_GRAD_SLICES fixed row slices; each slice's partial sum
// is formed by one thread in row order and the slices are added in slice order by one final launch: no atomics, equal
// inputs give equal bits.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "fsmn.h"
#include "grad_gemm.cuh"

namespace wekws {

namespace {

// ---------------------------------------------------------------------------------------------------- parameter pack
__global__ void fsmn_pack_kernel(const FsmnPackArgs a) {
  const FsmnParamCopy& p = a.p[blockIdx.y];
  const long long n = (long long)p.rows * p.cols;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(e / p.cols), c = (int)(e - (long long)r * p.cols);
    a.packed[p.dst + (long long)c * p.ld + r] = __ldg(p.src + e);
  }
}

// ---------------------------------------------------------------------------------------------------- memory block
// Training caches are empty, so cat = [zeros(pad) | p] with pad = lo - 1 + ro, and
//   m[t] = p[t - ro] + sum_i wl[i] p[t + i - pad] + sum_j wr[j] p[t + lo + j - pad]     (p = 0 outside [0, T)).
// With G = dL/dm of the same utterance (0 outside [0, T)):
//   dp[s]     = G[s + ro] + sum_i wl[i] G[s + pad - i] + sum_j wr[j] G[s + pad - lo - j]
//   dwl[c][i] = sum_{b,t} G[t] p[t + i - pad],   dwr[c][j] = sum_{b,t} G[t] p[t + lo + j - pad].
// CTA = 32 channels x 8 row groups over one of the FSMN_GRAD_SLICES row slices; each row group sums its contiguous
// share of the slice in row order, the eight are added in group order: the tap partials of the slice, in the
// parameters' [proj][order] layout.
constexpr int MB_C = 32, MB_R = 8;

struct MemArgs {
  const float* G; const float* p; const float* taps;   // taps: the pack's [lo + ro][P]
  float* dp; float* dwl_part; float* dwr_part;          // partials: + z * P * lo, + z * P * ro
  int M, T, P, lo, ro, rslice;
};

__global__ void __launch_bounds__(MB_C * MB_R) fsmn_grad_memory_kernel(const MemArgs a) {
  __shared__ float red[MB_R][MB_C][FSMN_MAX_TAPS + 1];
  const int cl = threadIdx.x & (MB_C - 1), rg = threadIdx.x / MB_C;
  const int c = blockIdx.x * MB_C + cl;
  const int lo = a.lo, ro = a.ro, pad = lo - 1 + ro, ntap = lo + ro, T = a.T, P = a.P;
  const int s_begin = blockIdx.y * a.rslice, s_end = min(a.M, s_begin + a.rslice);
  const int per = (a.rslice + MB_R - 1) / MB_R;
  const int r_begin = s_begin + rg * per, r_end = min(s_end, r_begin + per);
  float acc[FSMN_MAX_TAPS];
#pragma unroll
  for (int i = 0; i < FSMN_MAX_TAPS; ++i) acc[i] = 0.f;
  if (c < P) {
    for (int r = r_begin; r < r_end; ++r) {
      const int t = r % T, base = r - t;
      auto G = [&](int u) -> float { return u >= 0 && u < T ? __ldg(a.G + (long long)(base + u) * P + c) : 0.f; };
      auto pv = [&](int u) -> float { return u >= 0 && u < T ? __ldg(a.p + (long long)(base + u) * P + c) : 0.f; };
      float d = G(t + ro);
      for (int i = 0; i < lo; ++i) d = fmaf(__ldg(a.taps + i * P + c), G(t + pad - i), d);
      for (int j = 0; j < ro; ++j) d = fmaf(__ldg(a.taps + (lo + j) * P + c), G(t + pad - lo - j), d);
      a.dp[(long long)r * P + c] = d;
      const float g = G(t);
#pragma unroll
      for (int i = 0; i < FSMN_MAX_TAPS; ++i)
        if (i < ntap) acc[i] = fmaf(g, pv(t + i - pad), acc[i]);   // cat[t + i], left taps then right
    }
  }
#pragma unroll
  for (int i = 0; i < FSMN_MAX_TAPS; ++i)
    if (i < ntap) red[rg][cl][i] = acc[i];
  __syncthreads();
  // thread (cl, rg) adds the eight groups' sums of taps rg, rg + 8, ... in group order
  if (c < P) {
    for (int i = rg; i < ntap; i += MB_R) {
      float s = 0.f;
      for (int q = 0; q < MB_R; ++q) s += red[q][cl][i];
      if (i < lo) a.dwl_part[(long long)blockIdx.y * P * lo + (long long)c * lo + i] = s;
      else a.dwr_part[(long long)blockIdx.y * P * ro + (long long)c * ro + (i - lo)] = s;
    }
  }
}

long long param_numel(const FsmnArgs& a, int idx) {
  // state_dict order: in_linear1 W, b; in_linear2 W, b; per layer Wp, wl, wr, Wa, ba; out_linear1 W, b; out_linear2 W, b
  const int D = a.lin, P = a.proj;
  if (idx < 4) {
    const long long n[4] = {(long long)a.aff_in * a.idim, a.aff_in, (long long)D * a.aff_in, D};
    return n[idx];
  }
  const int k = idx - 4;
  if (k < 5 * a.L) {
    const long long n[5] = {(long long)P * D, (long long)P * a.lorder, (long long)P * a.rorder, (long long)D * P, D};
    return n[k % 5];
  }
  const long long n[4] = {(long long)a.aff_out * D, a.aff_out, (long long)a.odim * a.aff_out, a.odim};
  return n[k - 5 * a.L];
}

int max_width(const FsmnArgs& a) {
  int w = a.aff_in > a.lin ? a.aff_in : a.lin;
  if (a.proj > w) w = a.proj;
  return a.aff_out > w ? a.aff_out : w;
}

}  // namespace

int fsmn_pack_launch(const FsmnPackArgs& a, cudaStream_t st) {
  WEKWS_REQUIRE(a.n >= 1 && a.n <= FSMN_MAX_PARAMS, "fsmn_pack_launch: %d parameters", a.n);
  long long most = 0;
  for (int i = 0; i < a.n; ++i) most = std::max(most, (long long)a.p[i].rows * a.p[i].cols);
  const int bx = (int)std::min<long long>((most + 255) / 256, 64);
  fsmn_pack_kernel<<<dim3(bx, a.n), 256, 0, st>>>(a);
  return check_launch("fsmn_pack_kernel");
}

int fsmn_backward_launches(int L) { return 8 + 5 * L; }

long long fsmn_backward_workspace_floats(const FsmnArgs& a, long long M) {
  long long parts = 0;
  for (int i = 0; i < 8 + 5 * a.L; ++i) parts += param_numel(a, i);
  return FSMN_GRAD_SLICES * parts + 2 * M * max_width(a);
}

// The chain, from the top: G5 = dL/dlogits (M x O), x5 = out_linear1 output, h_l = input of FSMN layer l (h_0 after
// in_linear2's ReLU, h_L the last layer's output), p_l / m_l its projection / memory-block output, x1 = in_linear1 out.
//   out_linear2:  dW, db from (G5, x5);       dx5 = G5 W_o2
//   out_linear1:  dW, db from (dx5, h_L);     dh_L = (dx5 W_o1) * [h_L > 0]
//   layer l = L-1 .. 0:
//     Affine:     dW, db from (dh_{l+1}, m_l);  dm = dh_{l+1} W_a
//     memory:     dp, dwl, dwr from (dm, p_l)
//     Linear:     dW from (dp, h_l);             dh_l = (dp W_p) * [h_l > 0]
//   in_linear2:   dW, db from (dh_0, x1);     dx1 = dh_0 W_i2
//   in_linear1:   dW, db from (dx1, CMVN(feats))
// then one launch adds the slices of every parameter.  Launches: (4 + 2 L) dW + (3 + 2 L) dX + L memory + 1 = 8 + 5 L.
// G5 is read by two GEMMs: the dX one (once per 64-column tile of out_linear1's width) and the dW one (once per
// 64-column tile of x5); its bias sum rides on the dW GEMM.
int fsmn_backward_launch(const FsmnArgs& a, const float* feats, const float* saved, const float* grad_out, int B, int T,
                         float* const* grads, float* ws, cudaStream_t st) {
  const long long M = (long long)B * T;
  WEKWS_REQUIRE(a.L >= 1 && a.L <= FSMN_MAX_LAYERS && a.lorder + a.rorder <= FSMN_MAX_TAPS,
                "fsmn backward: %d layers, %d + %d taps unsupported", a.L, a.lorder, a.rorder);
  WEKWS_REQUIRE(M >= 1 && M < (1LL << 31) / max_width(a), "fsmn backward: %lld frames unsupported", M);
  const int nparam = 8 + 5 * a.L;
  const int S = FSMN_GRAD_SLICES;
  const int kslice = (int)((M + S - 1) / S);
  // workspace: the slice partials of every parameter in parameter order, then two (M, max width) gradient buffers
  std::vector<float*> part(nparam);
  float* w = ws;
  for (int i = 0; i < nparam; ++i) { part[i] = w; w += S * param_numel(a, i); }
  float* buf[2] = {w, w + M * max_width(a)};
  const float* W = a.w;
  auto sv = [&](int which, int l) { return saved + fsmn_saved_offset(a, M, which, l); };
  int rc;
  // dW (and db) of a Linear N <- K from dY (M x N) and X (M x K)
  auto dW = [&](const float* dY, int N, const float* X, int K, int pw, int pb, const float* mean, const float* scale) {
    GemmArgs g{};
    g.A = dY; g.sai = 1; g.sak = N;
    g.B = X; g.sbk = K; g.sbj = 1; g.bmean = mean; g.bscale = scale;
    g.C = part[pw]; g.ldc = K; g.c_slice = (long long)N * K;
    g.bias_out = pb >= 0 ? part[pb] : nullptr; g.bias_slice = N;
    g.I = N; g.J = K; g.K = (int)M; g.kslice = kslice;
    return gemm(g, S, st);
  };
  // dX (M x K) = dY (M x N) W, W from the pack's W^T [K][Npad]; masked by [mask > 0] if given
  auto dX = [&](const float* dY, int N, int w_off, int Npad, int K, float* out, const float* mask) {
    GemmArgs g{};
    g.A = dY; g.sai = N; g.sak = 1;
    g.B = W + w_off; g.sbk = 1; g.sbj = Npad;
    g.C = out; g.ldc = K; g.mask = mask; g.ldm = K;
    g.I = (int)M; g.J = K; g.K = N; g.kslice = N;
    return gemm(g, 1, st);
  };
  const int D = a.lin, P = a.proj, L = a.L;
  const int pi = 4 + 5 * L;                      // index of out_linear1.weight
  // out_linear2, out_linear1
  if ((rc = dW(grad_out, a.odim, sv(5, 0), a.aff_out, pi + 2, pi + 3, nullptr, nullptr))) return rc;
  if ((rc = dX(grad_out, a.odim, a.o_w_out2, a.np_odim, a.aff_out, buf[0], nullptr))) return rc;
  const float* hL = L > 0 ? sv(4, L - 1) : sv(1, 0);
  if ((rc = dW(buf[0], a.aff_out, hL, D, pi, pi + 1, nullptr, nullptr))) return rc;
  if ((rc = dX(buf[0], a.aff_out, a.o_w_out1, a.np_aff_out, D, buf[1], hL))) return rc;
  // FSMN layers: dh_{l+1} in buf[1]
  for (int l = L - 1; l >= 0; --l) {
    const int lw = a.o_layers + l * a.layer_stride, q = 4 + 5 * l;
    const float* h_in = l > 0 ? sv(4, l - 1) : sv(1, 0);
    if ((rc = dW(buf[1], D, sv(3, l), P, q + 3, q + 4, nullptr, nullptr))) return rc;
    if ((rc = dX(buf[1], D, lw + a.lo_wa, a.np_lin, P, buf[0], nullptr))) return rc;           // dm -> buf[0]
    MemArgs m{};
    m.G = buf[0]; m.p = sv(2, l); m.taps = W + lw + a.lo_taps;
    m.dp = buf[1]; m.dwl_part = part[q + 1]; m.dwr_part = part[q + 2];                         // dp -> buf[1]
    m.M = (int)M; m.T = T; m.P = P; m.lo = a.lorder; m.ro = a.rorder; m.rslice = kslice;
    fsmn_grad_memory_kernel<<<dim3((P + MB_C - 1) / MB_C, S), MB_C * MB_R, 0, st>>>(m);
    if ((rc = check_launch("fsmn_grad_memory_kernel"))) return rc;
    if ((rc = dW(buf[1], P, h_in, D, q, -1, nullptr, nullptr))) return rc;
    if ((rc = dX(buf[1], P, lw + a.lo_wp, a.np_proj, D, buf[0], h_in))) return rc;             // dh_l -> buf[0]
    std::swap(buf[0], buf[1]);                                                                 // dh_l in buf[1]
  }
  // in_linear2, in_linear1 (the latter against the CMVN-normalised features, recomputed on load)
  if ((rc = dW(buf[1], D, sv(0, 0), a.aff_in, 2, 3, nullptr, nullptr))) return rc;
  if ((rc = dX(buf[1], D, a.o_w_in2, a.np_lin, a.aff_in, buf[0], nullptr))) return rc;
  const float* mean = a.has_cmvn ? W + a.o_mean : nullptr;
  if ((rc = dW(buf[0], a.aff_in, feats, a.idim, 0, 1, mean, W + a.o_istd))) return rc;
  // slice sums into the caller's gradients
  ReduceArgs r{};
  r.njobs = nparam;
  for (int i = 0; i < nparam; ++i) {
    r.j[i].part = part[i]; r.j[i].out = grads[i]; r.j[i].n = param_numel(a, i);
  }
  return reduce_slices(r, st);
}

}  // namespace wekws
