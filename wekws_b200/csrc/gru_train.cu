// GRU training (wekws/utils/executor.py Executor.train with examples/hi_xiaowen/s0/conf/gru.yaml): the backward of the
// storing forward (gru.cu, gru_launch with save) to every parameter of the reference's GRU model: the preprocessing
// Linear, each layer of torch.nn.GRU and the linear classifier.
//
// FP32 FMA throughout, as the forward.  Rows are the M = B * T frames, padding included, as torch's autograd takes
// them.  Per layer, from the top, with dh the gradient of the layer's output h_t:
//   dn = dh (1 - z), dz = dh (h_{t-1} - n), da_n = dn (1 - n^2), dr = da_n hn, da_r = dr r (1 - r), da_z = dz z (1 - z)
//   dgi = [da_r, da_z, da_n], dgh = [da_r, da_z, da_n r], dh_{t-1} += dh z + W_hh^T dgh
// (hn = W_hn h_{t-1} + b_hn, kept by the forward).  The reverse recurrence is one sequential kernel per layer
// (gru_bptt_kernel, W_hh resident in shared memory); everything else is a GEMM over all M rows (grad_gemm.cuh):
// dX = dgi W_ih (the layer below's output gradient, for layer 0 masked by the ReLU), dW_ih = dgi^T X,
// dW_hh = dgh^T H_{t-1}, the biases as column sums.  Weight gradients are summed over FSMN_GRAD_SLICES fixed row slices
// and the slices added in order: no atomics, equal inputs give equal bits.
#include <vector>

#include "common.cuh"
#include "grad_gemm.cuh"
#include "gru.h"

namespace wekws {

namespace {

constexpr int GH = 128, GG = 3 * GH;
constexpr int WLD = GH + 1;        // row stride of W_hh in shared memory: conflict-free fill along g and reads along k

// dL/d(pre-activation logits): g y (1 - y) for Sigmoid (torch's sigmoid_backward order), g for Identity
__global__ void gru_grad_logits_kernel(const float* g, const float* y, float* d, long long n, int sigmoid) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const float gv = __ldg(g + e);
    if (sigmoid) {
      const float yv = __ldg(y + e);
      d[e] = gv * (1.f - yv) * yv;
    } else {
      d[e] = gv;
    }
  }
}

struct BpttArgs {
  const float* w;          // the layer's block of the pack: row k = [W_ih[:, k] | W_hh[:, k]] (gru.cu)
  const float* dh_in;      // (M, H): the gradient of h_t from above (classifier or the next layer)
  const float* hs; const float* rs; const float* zs; const float* ns; const float* hns;   // the layer's saved blocks
  float* dgi; float* dgh;  // (M, G)
  float* hprev;            // (M, H): h_{t-1} (0 at t = 0), the B operand of dW_hh
  int B, T, n_tiles;
};

// A CTA owns S streams for all T steps, one thread per gate row (3H = 384).  Per step: each (stream, unit) element
// forms its gate gradients from dh = dh_in + the carry and stores dgi / dgh / h_{t-1}; then thread (k, part) sums
// W_hh[g][k] dgh[g] over the gates g of its third; the next step adds the three thirds to dh z.  Each step's rows
// are loaded into registers one step ahead.
template <int S>
__global__ void __launch_bounds__(GG, 1) gru_bptt_kernel(const BpttArgs a) {
  extern __shared__ __align__(16) float sm[];
  float* W = sm;                         // [G][WLD]
  float* dg = W + GG * WLD;              // [S][G]  this step's dgh
  float* red = dg + S * GG;              // [3][S][H]  the thirds of W_hh^T dgh
  float* cz = red + 3 * S * GH;          // [S][H]  dh z
  constexpr int NE = (S * GH + GG - 1) / GG;
  const int tid = threadIdx.x;
  const long long T = a.T;
  for (int e = tid; e < GG * GH; e += GG) {
    const int k = e / GG, g = e - k * GG;
    W[g * WLD + k] = __ldg(a.w + (long long)k * 2 * GG + GG + g);
  }
  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    const int b0 = tile * S, Sv = min(S, a.B - b0);
    __syncthreads();                     // W filled; the previous tile's last step done
    for (int i = tid; i < S * GH; i += GG) {
      cz[i] = 0.f;
      red[i] = 0.f; red[S * GH + i] = 0.f; red[2 * S * GH + i] = 0.f;
    }
    float n_dh[NE], n_r[NE], n_z[NE], n_n[NE], n_hn[NE], n_hp[NE];
#define GRU_BPTT_LOAD(tt)                                                                             \
  _Pragma("unroll") for (int q = 0; q < NE; ++q) {                                                    \
    const int i = tid + q * GG, s = i / GH, j = i - s * GH;                                           \
    n_dh[q] = n_r[q] = n_z[q] = n_n[q] = n_hn[q] = n_hp[q] = 0.f;                                     \
    if (i < S * GH && s < Sv) {                                                                       \
      const long long o = ((b0 + s) * T + (tt)) * GH + j;                                             \
      n_dh[q] = __ldg(a.dh_in + o); n_r[q] = __ldg(a.rs + o); n_z[q] = __ldg(a.zs + o);               \
      n_n[q] = __ldg(a.ns + o); n_hn[q] = __ldg(a.hns + o);                                           \
      n_hp[q] = (tt) > 0 ? __ldg(a.hs + o - GH) : 0.f;                                                \
    }                                                                                                 \
  }
    GRU_BPTT_LOAD(T - 1)
    __syncthreads();
    for (long long t = T - 1; t >= 0; --t) {
      float c_dh[NE], c_r[NE], c_z[NE], c_n[NE], c_hn[NE], c_hp[NE];
#pragma unroll
      for (int q = 0; q < NE; ++q) {
        c_dh[q] = n_dh[q]; c_r[q] = n_r[q]; c_z[q] = n_z[q]; c_n[q] = n_n[q]; c_hn[q] = n_hn[q]; c_hp[q] = n_hp[q];
      }
      if (t > 0) { GRU_BPTT_LOAD(t - 1) }
#pragma unroll
      for (int q = 0; q < NE; ++q) {
        const int i = tid + q * GG, s = i / GH, j = i - s * GH;
        if (i < S * GH) {
          const float carry = ((cz[i] + red[i]) + red[S * GH + i]) + red[2 * S * GH + i];
          const float dh = c_dh[q] + carry;
          const float r = c_r[q], z = c_z[q], n = c_n[q];
          const float dn = dh * (1.f - z);
          const float dz = dh * (c_hp[q] - n);
          const float dan = dn * (1.f - n * n);
          const float dar = dan * c_hn[q] * (r * (1.f - r));
          const float daz = dz * (z * (1.f - z));
          const float danr = dan * r;
          const bool live = s < Sv;
          dg[s * GG + j] = live ? dar : 0.f;
          dg[s * GG + GH + j] = live ? daz : 0.f;
          dg[s * GG + 2 * GH + j] = live ? danr : 0.f;
          cz[i] = live ? dh * z : 0.f;
          if (live) {
            const long long row = (b0 + s) * T + t;
            float* gi = a.dgi + row * GG + j;
            float* gh = a.dgh + row * GG + j;
            gi[0] = dar; gi[GH] = daz; gi[2 * GH] = dan;
            gh[0] = dar; gh[GH] = daz; gh[2 * GH] = danr;
            a.hprev[row * GH + j] = c_hp[q];
          }
        }
      }
      __syncthreads();
      {
        const int k = tid & (GH - 1), part = tid >> 7;
        const float* w = W + part * GH * WLD + k;
        const float* d = dg + part * GH;
        float acc[S];
#pragma unroll
        for (int s = 0; s < S; ++s) acc[s] = 0.f;
#pragma unroll 4
        for (int g = 0; g < GH; g += 4) {
          const float w0 = w[g * WLD], w1 = w[(g + 1) * WLD], w2 = w[(g + 2) * WLD], w3 = w[(g + 3) * WLD];
#pragma unroll
          for (int s = 0; s < S; ++s) {
            const float4 d4 = *reinterpret_cast<const float4*>(d + s * GG + g);
            acc[s] = fmaf(w0, d4.x, acc[s]); acc[s] = fmaf(w1, d4.y, acc[s]);
            acc[s] = fmaf(w2, d4.z, acc[s]); acc[s] = fmaf(w3, d4.w, acc[s]);
          }
        }
#pragma unroll
        for (int s = 0; s < S; ++s) red[(part * S + s) * GH + k] = acc[s];
      }
      __syncthreads();
    }
#undef GRU_BPTT_LOAD
  }
}

template <int S>
int bptt_s(BpttArgs a, cudaStream_t st) {
  a.n_tiles = (a.B + S - 1) / S;
  const size_t smem = (size_t)(GG * WLD + S * (GG + 3 * GH + GH)) * sizeof(float);
  if (const int rc = opt_in_smem((const void*)gru_bptt_kernel<S>, smem)) return rc;
  const int sms = device_sm_count();
  gru_bptt_kernel<S><<<a.n_tiles < sms ? a.n_tiles : sms, GG, smem, st>>>(a);
  return check_launch("gru_bptt_kernel");
}

// streams per CTA as the forward takes them (gru.cu gru_launch): one wave of CTAs
int bptt_launch(const BpttArgs& a, cudaStream_t st) {
  const int sms = device_sm_count();
  const int S = a.B <= sms ? 1 : a.B <= 2 * sms ? 2 : a.B <= 4 * sms ? 4 : 8;
  switch (S) {
    case 1: return bptt_s<1>(a, st);
    case 2: return bptt_s<2>(a, st);
    case 4: return bptt_s<4>(a, st);
    default: return bptt_s<8>(a, st);
  }
}

// elements of parameter idx in named_parameters order (gru_num_params)
long long param_numel(const GruArgs& a, int idx) {
  const long long H = a.H, G = 3 * H;
  if (idx < 2) return idx == 0 ? H * a.idim : H;
  const int k = idx - 2;
  if (k < 4 * a.L) return k % 4 < 2 ? G * H : G;
  return k == 4 * a.L ? (long long)a.odim * H : a.odim;
}

}  // namespace

int gru_num_params(int L) { return 4 + 4 * L; }
int gru_backward_launches(int L) { return 5 + 4 * L; }

long long gru_backward_workspace_floats(const GruArgs& a, long long M) {
  long long parts = 0;
  for (int i = 0; i < gru_num_params(a.L); ++i) parts += param_numel(a, i);
  return FSMN_GRAD_SLICES * parts + M * (8LL * a.H + a.odim);
}

// The chain, from the top (launches: 1 + 2 + 4 L + 2 = 5 + 4 L):
//   dlogit = dL/dout through the activation;  classifier: dW, db from (dlogit, h of layer L-1);  dh = dlogit W_c
//   layer l = L-1 .. 0:  the reverse recurrence -> dgi, dgh, h_{t-1};  dW_ih, db_ih from (dgi, X_l);
//                        dW_hh, db_hh from (dgh, h_{t-1});  dX_l = dgi W_ih (layer 0: masked by x0 > 0)
//   preprocessing:       dW, db from (dX_0, CMVN(feats))
// then one launch adds the slices of every parameter.
int gru_backward_launch(const GruArgs& a, const float* feats, const float* saved, const float* out,
                        const float* grad_out, int B, int T, float* const* grads, float* ws, cudaStream_t st) {
  const long long M = (long long)B * T;
  const int H = a.H, G = 3 * H, L = a.L, O = a.odim;
  WEKWS_REQUIRE(H == GH && L >= 1 && L <= 4, "gru backward: hidden %d, %d layers unsupported", H, L);
  WEKWS_REQUIRE(M >= 1 && M < (1LL << 31), "gru backward: %lld frames unsupported", M);
  const int nparam = gru_num_params(L);
  const int S = FSMN_GRAD_SLICES;
  const int kslice = (int)((M + S - 1) / S);
  // workspace: the slice partials of every parameter in parameter order, then dh (M, H), dgi, dgh (M, G),
  // h_{t-1} (M, H), dlogit (M, O)
  std::vector<float*> part(nparam);
  float* w = ws;
  for (int i = 0; i < nparam; ++i) { part[i] = w; w += S * param_numel(a, i); }
  float* dh = w;
  float* dgi = dh + M * H;
  float* dgh = dgi + M * G;
  float* hprev = dgh + M * G;
  float* dlogit = hprev + M * H;
  const float* V = a.vec;
  auto blk = [&](int l, int which) { return saved + gru_saved_block(M, H, l, which); };
  int rc;
  auto dW = [&](const float* dY, int N, const float* X, int K, int pw, int pb, const float* mean, const float* scale) {
    GemmArgs g{};
    g.A = dY; g.sai = 1; g.sak = N;
    g.B = X; g.sbk = K; g.sbj = 1; g.bmean = mean; g.bscale = scale;
    g.C = part[pw]; g.ldc = K; g.c_slice = (long long)N * K;
    g.bias_out = part[pb]; g.bias_slice = N;
    g.I = N; g.J = K; g.K = (int)M; g.kslice = kslice;
    return gemm(g, S, st);
  };
  // dX (M x K) = dY (M x N) W, W^T [K][ld] read from the pack at w_off; masked by [mask > 0] if given
  auto dX = [&](const float* dY, int N, long long w_off, int ld, int K, float* dst, const float* mask) {
    GemmArgs g{};
    g.A = dY; g.sai = N; g.sak = 1;
    g.B = V + w_off; g.sbk = 1; g.sbj = ld;
    g.C = dst; g.ldc = K; g.mask = mask; g.ldm = K;
    g.I = (int)M; g.J = K; g.K = N; g.kslice = N;
    return gemm(g, 1, st);
  };
  {
    const long long n = M * O;
    const int bx = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
    gru_grad_logits_kernel<<<bx, 256, 0, st>>>(grad_out, out, dlogit, n, a.act == WEKWS_ACT_SIGMOID);
    if ((rc = check_launch("gru_grad_logits_kernel"))) return rc;
  }
  const int pc = 2 + 4 * L;                      // index of classifier.linear.weight
  if ((rc = dW(dlogit, O, blk(L - 1, 0), H, pc, pc + 1, nullptr, nullptr))) return rc;
  if ((rc = dX(dlogit, O, a.v_wc, O, H, dh, nullptr))) return rc;
  for (int l = L - 1; l >= 0; --l) {
    const long long lw = a.v_layers + (long long)l * a.v_layer_stride;
    BpttArgs r{};
    r.w = V + lw; r.dh_in = dh;
    r.hs = blk(l, 0); r.rs = blk(l, 1); r.zs = blk(l, 2); r.ns = blk(l, 3); r.hns = blk(l, 4);
    r.dgi = dgi; r.dgh = dgh; r.hprev = hprev;
    r.B = B; r.T = T;
    if ((rc = bptt_launch(r, st))) return rc;
    const float* X = l > 0 ? blk(l - 1, 0) : saved;        // layer l's input: the layer below's h, or x0
    const int q = 2 + 4 * l;
    if ((rc = dW(dgi, G, X, H, q, q + 2, nullptr, nullptr))) return rc;
    if ((rc = dW(dgh, G, hprev, H, q + 1, q + 3, nullptr, nullptr))) return rc;
    if ((rc = dX(dgi, G, lw, 2 * G, H, dh, l > 0 ? nullptr : saved))) return rc;
  }
  const float* mean = a.has_cmvn ? V + a.v_mean : nullptr;
  if ((rc = dW(dh, H, feats, a.idim, 0, 1, mean, V + a.v_istd))) return rc;
  ReduceArgs red{};
  red.njobs = nparam;
  for (int i = 0; i < nparam; ++i) {
    red.j[i].part = part[i]; red.j[i].out = grads[i]; red.j[i].n = param_numel(a, i);
  }
  return reduce_slices(red, st);
}

}  // namespace wekws
