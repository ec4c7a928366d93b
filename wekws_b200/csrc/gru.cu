// Fused KWSModel.forward for the GRU backbone (reference wekws/model/kws_model.py:128-133:
// torch.nn.GRU(hdim, hdim, num_layers, batch_first=True) between LinearSubsampling1
// subsampling.py:53-57 and LinearClassifier classifier.py:63-67).
//
// PyTorch gate order r, z, n:  r = s(W_ir x + b_ir + W_hr h + b_hr), z likewise,
// n = tanh(W_in x + b_in + r * (W_hn h + b_hn)),  h' = (1 - z) * n + z * h.
//
// A CTA owns S streams for the whole chunk of T frames; hidden state, layer input and gate
// pre-activations stay in shared memory across time steps and layers, so per step only the idim
// input features are read and odim posteriors written; the (L,B,H) cache is read and written once.
// One thread per gate row (3H = 384 threads).  The weights (786 KB for 2 layers) do not fit on chip,
// so every step streams them from L2 through a double-buffered shared-memory ring of 48 KB chunks
// (16 k-rows of [W_ih | W_hh], one cp.async.bulk each, mbarrier-signalled): the TMA engine keeps
// ~96 KB in flight per SM, which is what hides the L2 latency -- register-staged loads could not.
//
// The training forward (SAVE) is the same kernel that also stores what the backward (gru_train.cu) reads: the layer-0
// input and, per layer and step, h_t, r, z, n and W_hn h_{t-1} + b_hn (GruArgs::saved).
#include "common.cuh"
#include "gru.h"
#include "tc_common.cuh"

namespace wekws {

namespace {

using namespace tc;

constexpr int GH = 128, GG = 3 * GH;
constexpr int KCH = 16;                          // k-rows per weight chunk
constexpr int CHUNK_FLOATS = KCH * 2 * GG;       // 12288 floats = 48 KB
constexpr int NCHUNK = GH / KCH;                 // 8 chunks per layer

template <int S, bool SAVE>
__global__ void __launch_bounds__(GG, 1) gru_kernel(const GruArgs a) {
  extern __shared__ __align__(128) float sm[];
  float* ring = sm;                               // [2][CHUNK_FLOATS]
  float* xin = ring + 2 * CHUNK_FLOATS;           // [S][H]   current layer input
  float* hst = xin + S * GH;                      // [L][S][H]
  float* gi = hst + a.L * S * GH;                 // [S][G]
  float* gh = gi + S * GG;                        // [S][G]
  float* fin = gh + S * GG;                       // [S][idimP]
  __shared__ uint64_t full[2];
  const int tid = threadIdx.x;
  const int idim = a.idim, idimP = (idim + 3) & ~3;
  const float* vec = a.vec;
  const long long M = (long long)a.B * a.T;        // rows of a saved block
  if (tid == 0) {
    mbar_init(&full[0], 1); mbar_init(&full[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  uint32_t seq_issued = 0, seq_used = 0;          // weight-chunk sequence numbers (slot = seq & 1)
  // chunk `c` of the per-step stream: layer l = c / NCHUNK, rows [KCH * (c % NCHUNK), +KCH)
  auto issue = [&](int c) {                       // thread 0
    const int l = c / NCHUNK, kc = c - l * NCHUNK;
    const float* src = vec + a.v_layers + (size_t)l * a.v_layer_stride + (size_t)kc * CHUNK_FLOATS;
    const uint32_t slot = seq_issued & 1;
    fence_proxy_async();                          // the slot was read through the generic proxy
    mbar_arrive_expect_tx(&full[slot], CHUNK_FLOATS * 4);
    bulk_g2s(ring + slot * CHUNK_FLOATS, src, CHUNK_FLOATS * 4, &full[slot]);
    ++seq_issued;
  };
  const int chunks_per_step = a.L * NCHUNK;

  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    const int b0 = tile * S;
    const int Sv = min(S, a.B - b0);
    __syncthreads();
    for (int i = tid; i < a.L * S * GH; i += GG) {
      const int l = i / (S * GH), rem = i - l * S * GH, s = rem / GH, j = rem - s * GH;
      float v = 0.f;
      if (a.in_cache != nullptr && s < Sv) v = a.in_cache[((size_t)l * a.B + b0 + s) * GH + j];
      hst[i] = v;
    }
    if (tid == 0) issue(0);                       // first chunk of the first step of this tile
    for (int t = 0; t < a.T; ++t) {
      // features of this step (+CMVN)
      for (int i = tid; i < S * idimP; i += GG) {
        const int s = i / idimP, k = i - s * idimP;
        float v = 0.f;
        if (s < Sv && k < idim) {
          v = __ldg(a.feats + ((size_t)(b0 + s) * a.T + t) * idim + k);
          if (a.has_cmvn) v = (v - __ldg(vec + a.v_mean + k)) * __ldg(vec + a.v_istd + k);
        }
        fin[i] = v;
      }
      __syncthreads();
      // preprocessing Linear + ReLU: all 384 threads, thread (j, part) sums every third k; partials through `gi`
      {
        const int j = tid & (GH - 1), part = tid >> 7;
        float acc[S];
#pragma unroll
        for (int s = 0; s < S; ++s) acc[s] = 0.f;
        const float* wp = vec + a.v_wp + j;             // WpT[k][H]
#pragma unroll 4
        for (int k = part; k < idim; k += 3) {
          const float w = __ldg(wp + k * GH);
#pragma unroll
          for (int s = 0; s < S; ++s) acc[s] = fmaf(w, fin[s * idimP + k], acc[s]);
        }
#pragma unroll
        for (int s = 0; s < S; ++s) gi[(part * S + s) * GH + j] = acc[s];
      }
      __syncthreads();
      for (int i = tid; i < S * GH; i += GG) {
        const int s = i / GH, j = i - s * GH;
        const float v = gi[s * GH + j] + gi[(S + s) * GH + j] + gi[(2 * S + s) * GH + j] + __ldg(vec + a.v_bp + j);
        xin[i] = fmaxf(v, 0.f);
        if constexpr (SAVE) {
          if (s < Sv) a.saved[((long long)(b0 + s) * a.T + t) * GH + j] = xin[i];
        }
      }
      __syncthreads();
      for (int l = 0; l < a.L; ++l) {
        const float* hl = hst + l * S * GH;
        float ai[S], ah[S];
        {
          const float* bias = vec + a.v_layers + (size_t)l * a.v_layer_stride + 2 * GH * GG;
          const float bi = __ldg(bias + tid), bh = __ldg(bias + GG + tid);
#pragma unroll
          for (int s = 0; s < S; ++s) { ai[s] = bi; ah[s] = bh; }
        }
        for (int kc = 0; kc < NCHUNK; ++kc) {
          const uint32_t slot = seq_used & 1;
          // prefetch the following chunk into the other slot (its previous reader finished before the last barrier)
          if (tid == 0) {
            const int c = l * NCHUNK + kc + 1;
            if (c < chunks_per_step) issue(c);
            else if (t + 1 < a.T) issue(0);           // first chunk of the next time step
          }
          mbar_wait(&full[slot], (seq_used >> 1) & 1);
          const float* w = ring + slot * CHUNK_FLOATS + tid;
#pragma unroll
          for (int k4 = 0; k4 < KCH; k4 += 4) {
            float wi[4], wh[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) { wi[u] = w[(k4 + u) * 2 * GG]; wh[u] = w[(k4 + u) * 2 * GG + GG]; }
            const int k = kc * KCH + k4;
#pragma unroll
            for (int s = 0; s < S; ++s) {
              const float4 x4 = *reinterpret_cast<const float4*>(xin + s * GH + k);
              const float4 h4 = *reinterpret_cast<const float4*>(hl + s * GH + k);
              ai[s] = fmaf(wi[0], x4.x, ai[s]); ai[s] = fmaf(wi[1], x4.y, ai[s]);
              ai[s] = fmaf(wi[2], x4.z, ai[s]); ai[s] = fmaf(wi[3], x4.w, ai[s]);
              ah[s] = fmaf(wh[0], h4.x, ah[s]); ah[s] = fmaf(wh[1], h4.y, ah[s]);
              ah[s] = fmaf(wh[2], h4.z, ah[s]); ah[s] = fmaf(wh[3], h4.w, ah[s]);
            }
          }
          ++seq_used;
          __syncthreads();                            // everyone done with this slot before it is refilled
        }
#pragma unroll
        for (int s = 0; s < S; ++s) { gi[s * GG + tid] = ai[s]; gh[s * GG + tid] = ah[s]; }
        __syncthreads();
        for (int i = tid; i < S * GH; i += GG) {
          const int s = i / GH, j = i - s * GH;
          const float r = sigmoidf_acc(gi[s * GG + j] + gh[s * GG + j]);
          const float z = sigmoidf_acc(gi[s * GG + GH + j] + gh[s * GG + GH + j]);
          const float n = tanhf(gi[s * GG + 2 * GH + j] + r * gh[s * GG + 2 * GH + j]);
          const float hp = hst[(l * S + s) * GH + j];
          const float hn = (1.f - z) * n + z * hp;
          hst[(l * S + s) * GH + j] = hn;
          xin[s * GH + j] = hn;
          if constexpr (SAVE) {
            if (s < Sv) {
              float* dst = a.saved + M * GH * (1 + 5 * l) + ((long long)(b0 + s) * a.T + t) * GH + j;
              dst[0] = hn;
              dst[M * GH] = r;
              dst[2 * M * GH] = z;
              dst[3 * M * GH] = n;
              dst[4 * M * GH] = gh[s * GG + 2 * GH + j];
            }
          }
        }
        __syncthreads();
      }
      // classifier on the top layer's h_t: one warp per (stream, output), lanes split k, shuffle reduction
      for (int o = tid >> 5; o < Sv * a.odim; o += GG / 32) {
        const int s = o / a.odim, j = o - s * a.odim, lane = tid & 31;
        const float* wc = vec + a.v_wc + j;            // WcT[k][odim]
        float acc = 0.f;
#pragma unroll
        for (int u = 0; u < GH / 32; ++u) {
          const int k = lane + 32 * u;
          acc = fmaf(__ldg(wc + k * a.odim), xin[s * GH + k], acc);
        }
#pragma unroll
        for (int sh = 16; sh > 0; sh >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sh);
        if (lane == 0) {
          acc += __ldg(vec + a.v_bc + j);
          if (a.act == WEKWS_ACT_SIGMOID) acc = sigmoidf_acc(acc);
          a.out[((size_t)(b0 + s) * a.T + t) * a.odim + j] = acc;
        }
      }
      // (the next step's feature load only touches `fin`; the barrier after it orders the reuse of xin)
    }
    __syncthreads();
    for (int i = tid; i < a.L * Sv * GH; i += GG) {
      const int l = i / (Sv * GH), rem = i - l * Sv * GH, s = rem / GH, j = rem - s * GH;
      a.out_cache[((size_t)l * a.B + b0 + s) * GH + j] = hst[(l * S + s) * GH + j];
    }
  }
}

template <int S, bool SAVE>
int launch_s(const GruArgs& a, cudaStream_t st) {
  GruArgs b = a;
  b.n_tiles = (a.B + S - 1) / S;
  const int idimP = (a.idim + 3) & ~3;
  const size_t smem = (size_t)(2 * CHUNK_FLOATS + S * GH + a.L * S * GH + 2 * S * GG + S * idimP) * sizeof(float);
  const int sms = device_sm_count();
  if (const int rc = opt_in_smem((const void*)gru_kernel<S, SAVE>, smem)) return rc;
  const int grid = b.n_tiles < sms ? b.n_tiles : sms;
  gru_kernel<S, SAVE><<<grid, GG, smem, st>>>(b);
  return check_launch(SAVE ? "gru_kernel<save>" : "gru_kernel");
}

}  // namespace

int gru_launch(const GruArgs& a, cudaStream_t st, bool save) {
  WEKWS_REQUIRE(a.H == 128, "GRU hidden_dim %d unsupported (128 only)", a.H);
  WEKWS_REQUIRE(a.L >= 1 && a.L <= 4, "GRU num_layers %d unsupported (1..4)", a.L);
  const int sms = device_sm_count();
  // streams per CTA: keep the grid within one wave
  const int S = a.B <= sms ? 1 : a.B <= 2 * sms ? 2 : a.B <= 4 * sms ? 4 : 8;
  WEKWS_REQUIRE(!save || (a.saved != nullptr && a.in_cache == nullptr), "gru_launch: bad training-forward arguments");
  switch (S) {
    case 1: return save ? launch_s<1, true>(a, st) : launch_s<1, false>(a, st);
    case 2: return save ? launch_s<2, true>(a, st) : launch_s<2, false>(a, st);
    case 4: return save ? launch_s<4, true>(a, st) : launch_s<4, false>(a, st);
    default: return save ? launch_s<8, true>(a, st) : launch_s<8, false>(a, st);
  }
}

}  // namespace wekws
