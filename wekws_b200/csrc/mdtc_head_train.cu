// MDTC training with the speech-command heads (wekws/model/classifier.py GlobalClassifier / LastClassifier around
// Sequential(Linear(C, 64), ReLU, Dropout(p), Linear(64, odim)), kws_model.py:175-190, in Executor.train).
//
// The backbone is mdtc_train.cu's, run through its host orchestration with odim = 0: its forward leaves the stack sum
// s (B, T, C), and its backward starts from the stack sum's gradient ds.  This file adds three kernels, FP32 with
// double accumulation where the head sums over frames or utterances, and no atomics (equal inputs give equal bits):
//   forward   one CTA per utterance: pool = mean over the T frames (global, padding included, as torch.mean) or frame
//             T - 1 (last); h = W1 pool + b1; hd = Dropout(relu(h)); y = W2 hd + b2.  Keeps pool and h for the backward.
//   backward  one CTA per utterance: dhd = g W2; dh = dhd * mask * scale * [h > 0]; dpool = dh W1; ds written in full
//             (dpool / T on every frame, or dpool on frame T - 1 and zeros elsewhere).  Keeps dh and hd.
//   weights   one thread per element of dW1, db1, dW2, db2: the sum over the utterances in utterance order, in double,
//             rounded once.
// The Dropout mask is recomputed from the seed in the backward, never stored.
#include <algorithm>

#include "common.cuh"
#include "mdtc_head_train.h"
#include "tcn_train.h"

namespace wekws {

namespace {

constexpr int NT = 256;
constexpr int W = MDTC_HEAD_WIDTH;

struct HeadFwdArgs {
  const float* s;                                     // (B, T, C) stack sum
  const float* W1; const float* b1; const float* W2; const float* b2;
  float* out;                                         // (B, odim)
  float* pool; float* h;                              // (B, C), (B, 64) pre-ReLU; nullptr: not kept
  int T, odim, last;
  uint64_t seed; uint32_t theta; float scale;
};

template <int C>
__global__ void __launch_bounds__(NT) mdtc_head_fwd_kernel(const HeadFwdArgs a) {
  constexpr int G = NT / C;
  __shared__ double red[G][C];
  __shared__ float pool[C], hd[W];
  const int b = blockIdx.x, tid = threadIdx.x, c = tid % C, g = tid / C;
  const float* s = a.s + (long long)b * a.T * C;
  if (a.last) {
    if (tid < C) pool[tid] = s[(long long)(a.T - 1) * C + tid];
  } else {                                            // frame groups in order, each in frame order
    double acc = 0.0;
    for (int t = g; t < a.T; t += G) acc += (double)s[(long long)t * C + c];
    red[g][c] = acc;
    __syncthreads();
    if (tid < C) {
      double sum = 0.0;
      for (int q = 0; q < G; ++q) sum += red[q][tid];
      pool[tid] = (float)(sum / (double)a.T);
    }
  }
  __syncthreads();
  if (a.pool != nullptr && tid < C) a.pool[(long long)b * C + tid] = pool[tid];
  if (tid < W) {
    float acc = a.b1[tid];
    for (int i = 0; i < C; ++i) acc = fmaf(__ldg(a.W1 + tid * C + i), pool[i], acc);
    if (a.h != nullptr) a.h[(long long)b * W + tid] = acc;
    const float r = fmaxf(acc, 0.f);
    hd[tid] = dropout_keep(a.seed, MDTC_HEAD_DROPOUT_LAYER, b, 0, tid, a.theta) ? r * a.scale : 0.f;
  }
  __syncthreads();
  for (int o = tid; o < a.odim; o += NT) {
    float acc = a.b2[o];
    for (int j = 0; j < W; ++j) acc = fmaf(__ldg(a.W2 + (long long)o * W + j), hd[j], acc);
    a.out[(long long)b * a.odim + o] = acc;
  }
}

struct HeadBwdArgs {
  const float* g;                                     // (B, odim) d logits
  const float* h;                                     // (B, 64) the forward's pre-ReLU h
  const float* W1; const float* W2;
  float* ds;                                          // (B, T, C)
  float* dh; float* hd;                               // (B, 64) each, for the weight sums
  int T, odim, last;
  uint64_t seed; uint32_t theta; float scale;
};

template <int C>
__global__ void __launch_bounds__(NT) mdtc_head_bwd_kernel(const HeadBwdArgs a) {
  __shared__ float dhs[W], dpool[C];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid < W) {
    const float hv = a.h[(long long)b * W + tid];
    const bool keep = dropout_keep(a.seed, MDTC_HEAD_DROPOUT_LAYER, b, 0, tid, a.theta);
    a.hd[(long long)b * W + tid] = keep ? fmaxf(hv, 0.f) * a.scale : 0.f;
    const float* g = a.g + (long long)b * a.odim;
    float acc = 0.f;
    for (int o = 0; o < a.odim; ++o) acc = fmaf(g[o], __ldg(a.W2 + (long long)o * W + tid), acc);
    const float d = keep && hv > 0.f ? acc * a.scale : 0.f;      // Dropout's backward, then ReLU's
    a.dh[(long long)b * W + tid] = d;
    dhs[tid] = d;
  }
  __syncthreads();
  if (tid < C) {
    float acc = 0.f;
    for (int j = 0; j < W; ++j) acc = fmaf(dhs[j], __ldg(a.W1 + j * C + tid), acc);
    dpool[tid] = a.last ? acc : acc / (float)a.T;
  }
  __syncthreads();
  float* ds = a.ds + (long long)b * a.T * C;
  const long long n = (long long)a.T * C;
  for (long long e = tid; e < n; e += NT) {
    const int t = (int)(e / C);
    ds[e] = !a.last || t == a.T - 1 ? dpool[e % C] : 0.f;
  }
}

struct HeadSumArgs {
  const float* pool; const float* dh; const float* hd; const float* g;
  float* dW1; float* db1; float* dW2; float* db2;
  int B, C, odim;
};

__global__ void mdtc_head_wsum_kernel(const HeadSumArgs a) {
  const int C = a.C, O = a.odim, B = a.B;
  const int n1 = W * C, n2 = n1 + W, n3 = n2 + O * W, n4 = n3 + O;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n4; e += gridDim.x * blockDim.x) {
    double s = 0.0;
    if (e < n1) {                                     // dW1[j][c] = Sigma_b dh[b][j] pool[b][c]
      const int j = e / C, c = e % C;
      for (int b = 0; b < B; ++b) s = fma((double)a.dh[(long long)b * W + j], (double)a.pool[(long long)b * C + c], s);
      a.dW1[e] = (float)s;
    } else if (e < n2) {                              // db1[j] = Sigma_b dh[b][j]
      const int j = e - n1;
      for (int b = 0; b < B; ++b) s += (double)a.dh[(long long)b * W + j];
      a.db1[j] = (float)s;
    } else if (e < n3) {                              // dW2[o][j] = Sigma_b g[b][o] hd[b][j]
      const int q = e - n2, o = q / W, j = q % W;
      for (int b = 0; b < B; ++b) s = fma((double)a.g[(long long)b * O + o], (double)a.hd[(long long)b * W + j], s);
      a.dW2[q] = (float)s;
    } else {                                          // db2[o] = Sigma_b g[b][o]
      const int o = e - n3;
      for (int b = 0; b < B; ++b) s += (double)a.g[(long long)b * O + o];
      a.db2[o] = (float)s;
    }
  }
}

// the head's parameters (and gradients) follow the backbone's 2 + 12 L
inline int head_param(const MdtcTrainDims& d, int k) { return 2 + 12 * d.L + k; }

}  // namespace

long long mdtc_head_train_saved_floats(const MdtcTrainDims& d, long long B, long long T) {
  return mdtc_train_saved_floats(d, B * T) + B * (d.C + W);
}

long long mdtc_head_train_workspace_bytes(const MdtcTrainDims& d, long long B, long long T, bool save) {
  return mdtc_train_workspace_bytes(d, B * T, save);
}

long long mdtc_head_backward_workspace_bytes(const MdtcTrainDims& d, long long B, long long T) {
  return mdtc_backward_workspace_bytes(d, B * T) + 4 * (B * T * d.C + 2 * B * W);
}

int mdtc_head_train_forward_launch(const MdtcTrainDims& d, const MdtcHead& h, const float* feats,
                                   const float* const* params, const float* cmvn_mean, const float* cmvn_istd,
                                   float* const* running, const double* bn, float* out, float* out_cache, float* saved,
                                   void* workspace, int B, int T, cudaStream_t st) {
  int rc = mdtc_train_forward_launch(d, feats, params, cmvn_mean, cmvn_istd, running, bn, nullptr, out_cache, saved,
                                     workspace, B, T, st);
  if (rc) return rc;
  const long long M = (long long)B * T;
  float* kept = saved ? saved + mdtc_train_saved_floats(d, M) : nullptr;   // [pool (B, C)][h (B, 64)]
  HeadFwdArgs a{};
  a.s = mdtc_train_stack_sum(d, M, saved, workspace);
  a.W1 = params[head_param(d, 0)]; a.b1 = params[head_param(d, 1)];
  a.W2 = params[head_param(d, 2)]; a.b2 = params[head_param(d, 3)];
  a.out = out;
  a.pool = kept;
  a.h = kept ? kept + (long long)B * d.C : nullptr;
  a.T = T; a.odim = h.odim; a.last = h.last;
  a.seed = h.seed; a.theta = h.theta; a.scale = h.scale;
  if (d.C == 64) mdtc_head_fwd_kernel<64><<<B, NT, 0, st>>>(a);
  else mdtc_head_fwd_kernel<32><<<B, NT, 0, st>>>(a);
  return check_launch("mdtc_head_fwd_kernel");
}

int mdtc_head_backward_launch(const MdtcTrainDims& d, const MdtcHead& h, const float* feats,
                              const float* const* params, const float* cmvn_mean, const float* cmvn_istd,
                              const float* saved, const float* grad_out, int B, int T, float* const* grads,
                              void* workspace, cudaStream_t st) {
  const long long M = (long long)B * T;
  const float* kept = saved + mdtc_train_saved_floats(d, M);
  // workspace: [the backbone backward's][ds (B, T, C)][dh (B, 64)][hd (B, 64)]
  float* ds = (float*)((char*)workspace + mdtc_backward_workspace_bytes(d, M));
  float* dh = ds + M * d.C;
  float* hd = dh + (long long)B * W;
  HeadBwdArgs a{};
  a.g = grad_out; a.h = kept + (long long)B * d.C;
  a.W1 = params[head_param(d, 0)]; a.W2 = params[head_param(d, 2)];
  a.ds = ds; a.dh = dh; a.hd = hd;
  a.T = T; a.odim = h.odim; a.last = h.last;
  a.seed = h.seed; a.theta = h.theta; a.scale = h.scale;
  if (d.C == 64) mdtc_head_bwd_kernel<64><<<B, NT, 0, st>>>(a);
  else mdtc_head_bwd_kernel<32><<<B, NT, 0, st>>>(a);
  int rc = check_launch("mdtc_head_bwd_kernel");
  if (rc) return rc;
  HeadSumArgs s{};
  s.pool = kept; s.dh = dh; s.hd = hd; s.g = grad_out;
  s.dW1 = grads[head_param(d, 0)]; s.db1 = grads[head_param(d, 1)];
  s.dW2 = grads[head_param(d, 2)]; s.db2 = grads[head_param(d, 3)];
  s.B = B; s.C = d.C; s.odim = h.odim;
  const long long n = (long long)W * d.C + W + (long long)h.odim * W + h.odim;
  mdtc_head_wsum_kernel<<<(int)std::min<long long>((n + 255) / 256, 1024), 256, 0, st>>>(s);
  if ((rc = check_launch("mdtc_head_wsum_kernel"))) return rc;
  return mdtc_backward_launch(d, feats, params, cmvn_mean, cmvn_istd, saved, ds, B, T, grads, workspace, st);
}

}  // namespace wekws
