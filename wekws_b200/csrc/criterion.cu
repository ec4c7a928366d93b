// Held-out loss and accuracy with the reference's training criteria (wekws/model/loss.py criterion(), as
// wekws/utils/executor.py Executor.cv / Executor.test call it): max_pooling, ce and ctc.
//   * max_pooling: one CTA per utterance, one warp per keyword column; the loss is folded in the reference's own
//     (i, j) order in float32, so it differs from the reference only by logf ulps.
//   * ce: one warp per row.
//   * ctc: one warp per (b, t) row writes the softmax normaliser (the only pass over the B*T*V logits), one CTA per
//     utterance runs torch's log-space alpha recurrence (one thread per extended-label state), and with validation
//     the prefix beam search of ctc_decode.cu decodes the same softmax formed on load, then one warp per utterance
//     computes the edit distance of the best hypothesis to the label.  Calculator's back-trace (loss.py:395-453) only
//     moves to a predecessor whose distance differs by the step's cost, and `cor` costs 0, so ins + sub + del along
//     it is the edit distance and `all` is the label length: the accuracy needs the distance only.
//   * criterion_reduce_kernel (one thread) folds the per-term values in a fixed order and writes loss and accuracy.
// NaN propagates as in torch (max / min / clamp / argmax keep it), which fmaxf / fminf would not.
//
// Training (Executor.train: loss.backward()): the *_train entry points run the same forward and keep what the
// gradient needs (max_pooling: the pooled values; ce: the counted rows; ctc: alpha, (B, T, 2 Lmax + 1)), and the
// *_backward entry points write d loss / d logits, every element of it, as upstream * (unit gradient), the gradient
// torch's autograd gives for loss.py:
//   * max_pooling: the pooled frame gets -1 / (p B) (keyword column) or +1 / ((1 - p) B) (others), split evenly over
//     the positions that tie after masked_fill and clamp; masked ties and ties outside the clamp's closed interval
//     count in the split and receive nothing.
//   * ce: (softmax - onehot) / count on the counted rows.
//   * ctc: (softmax - occupancy) / B on the frames of a feasible utterance, NaN on those of an infeasible one, zero
//     on padding.  ctc_beta_kernel turns alpha into occupancies in place (one owner state per token, so the gradient
//     kernel needs no atomics), ctc_grad_kernel streams the logits once and the gradient once.
#include <math.h>

#include "common.cuh"
#include "ctc_decode.h"

namespace wekws {
namespace {

constexpr int kAccScoreBeam = 3, kAccPathBeam = 5;   // acc_utterance: ctc_prefix_beam_search(score, len, None, 3, 5)
constexpr int kMaxStates = 2 * WEKWS_CRITERION_MAX_LABEL + 1;
static_assert(kMaxStates <= 1024, "one thread per extended-label state");
constexpr int kIgnoreIndex = -100;                   // F.cross_entropy's ignore_index

enum Kind { kMaxPooling = 0, kCe = 1, kCtc = 2 };

__device__ __forceinline__ float max_nan(float a, float b) { return (a != a || a > b) ? a : b; }
__device__ __forceinline__ float min_nan(float a, float b) { return (a != a || a < b) ? a : b; }
__device__ __forceinline__ float clamp_nan(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }
// does (v, i) win over (bv, bi) in torch's arg-max: NaN first, then the larger value, then the lower index
__device__ __forceinline__ bool argmax_wins(float v, int i, float bv, int bi) {
  if (i < 0) return false;
  if (bi < 0) return true;
  const bool vn = v != v, bn = bv != bv;
  if (vn != bn) return vn;
  if (!vn && v != bv) return v > bv;
  return i < bi;
}

// max_pooling_loss (loss.py:44-87).  term[b][j]: -log(max) of the keyword column j == target, -log(min(1 - p)) of the
// others; correct[b]: the accuracy rule on the masked max over T then the first-index max over D.
// kTrain: pooled[b][j] keeps the pooled value for max_pool_grad_kernel.
template <bool kTrain>
__global__ void max_pool_kernel(const float* __restrict__ x, const int32_t* __restrict__ target,
                                const int32_t* __restrict__ lens, int T, int D, int min_duration,
                                float* __restrict__ term, int32_t* __restrict__ correct,
                                float* __restrict__ pooled) {
  extern __shared__ float colmax[];              // (D) masked max over T of each column
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const long long b = blockIdx.x;
  const int len = lens[b], tgt = target[b];
  const float* xb = x + b * (long long)T * D;
  for (int j = warp; j < D; j += nw) {
    const bool kw = j == tgt;
    float pool = kw ? -INFINITY : INFINITY, cmax = -INFINITY;
    for (int t = lane; t < T; t += 32) {
      const float v = xb[(long long)t * D + j];
      const bool pad = t >= len;
      cmax = max_nan(cmax, pad ? 0.f : v);
      if (kw) pool = max_nan(pool, clamp_nan(pad || t < min_duration ? 0.f : v, 1e-8f, 1.f));
      else pool = min_nan(pool, clamp_nan(pad ? 1.f : 1.f - v, 1e-8f, 1.f));
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float oc = __shfl_xor_sync(0xffffffffu, cmax, o), op = __shfl_xor_sync(0xffffffffu, pool, o);
      cmax = max_nan(cmax, oc);
      pool = kw ? max_nan(pool, op) : min_nan(pool, op);
    }
    if (lane == 0) {
      term[b * D + j] = -logf(pool);
      if constexpr (kTrain) pooled[b * D + j] = pool;
      colmax[j] = cmax;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float best = colmax[0];
    int idx = 0;
    for (int j = 1; j < D; ++j)
      if (argmax_wins(colmax[j], j, best, idx)) { best = colmax[j]; idx = j; }
    correct[b] = (best > 0.5f && idx == tgt) || (best < 0.5f && tgt < 0);
  }
}

// cross_entropy (loss.py:167-180): term[b] = -log_softmax(x[b])[target[b]] (unset for ignore_index), correct[b] =
// first-index argmax == target
__global__ void ce_kernel(const float* __restrict__ x, const int32_t* __restrict__ target, long long B, int C,
                          float* __restrict__ term, int32_t* __restrict__ correct) {
  const long long b = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  const float* p = x + b * C;
  float m, s;
  warp_row_max_sum(p, C, lane, m, s);
  float bv = 0.f;
  int bi = -1;
  for (int i = lane; i < C; i += 32) {
    const float v = p[i];
    if (argmax_wins(v, i, bv, bi)) { bv = v; bi = i; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_wins(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) {
    const int t = target[b];
    if (t != kIgnoreIndex) term[b] = -((p[t] - m) - logf(s));
    correct[b] = bi == t;
  }
}

// the softmax normaliser of every (b, t) row with t < lens[b]; padding rows feed neither the loss nor the decode
__global__ void ctc_row_kernel(const float* __restrict__ x, const int32_t* __restrict__ lens, long long B, long long T,
                               int V, float* __restrict__ row_max, float* __restrict__ row_sum) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B * T) return;
  const long long b = row / T;
  if (row - b * T >= lens[b]) return;
  const int lane = threadIdx.x & 31;
  float m, s;
  warp_row_max_sum(x + row * V, V, lane, m, s);
  if (lane == 0) {
    row_max[row] = m;
    row_sum[row] = s;
  }
}

// first token of label b: padded rows, or (label_stride == 0) labels back to back
__device__ __forceinline__ const int32_t* label_of(const int32_t* labels, long long label_stride,
                                                   const int32_t* label_lens, long long b) {
  if (label_stride > 0) return labels + b * label_stride;
  long long off = 0;
  for (long long k = 0; k < b; ++k) off += label_lens[k];
  return labels + off;
}

// F.ctc_loss of one utterance (blank 0, zero_infinity=False): torch's CPU recurrence (LossCTC.cpp), in float32.
// Thread s is extended-label state s of l' = (blank, l1, blank, l2, ..., blank); alpha is double-buffered in shared
// memory with one barrier per frame, and frame t + 1's log-probability is gathered before that barrier.
// kTrain: alpha[t][s] of the utterance's frames and states is also stored, (B, T, alpha_stride), for ctc_beta_kernel.
template <bool kTrain>
__global__ void ctc_alpha_kernel(const float* __restrict__ x, const float* __restrict__ row_max,
                                 const float* __restrict__ row_sum, const int32_t* __restrict__ lens,
                                 const int32_t* __restrict__ labels, long long label_stride,
                                 const int32_t* __restrict__ label_lens, long long T, int V,
                                 float* __restrict__ utt_loss, float* __restrict__ alpha_out, int alpha_stride) {
  extern __shared__ float alpha[];               // [2][blockDim.x]
  const int s = threadIdx.x, ns = blockDim.x;
  const long long b = blockIdx.x;
  const int n = lens[b], L = label_lens[b], S = 2 * L + 1;
  if (n == 0) {                                  // no frame: an empty label costs nothing, any other is infeasible
    if (s == 0) utt_loss[b] = L == 0 ? 0.f : INFINITY;
    return;
  }
  const int32_t* lab = label_of(labels, label_stride, label_lens, b);
  const bool active = s < S;
  const int tok = (active && (s & 1)) ? lab[s >> 1] : 0;
  const bool skip = active && (s & 1) && s >= 3 && lab[s >> 1] != lab[(s >> 1) - 1];   // l'_s != l'_{s-2}
  const float* xb = x + b * T * V;
  const float* mb = row_max + b * T;
  const float* sb = row_sum + b * T;
  auto log_prob = [&](int t) { return (__ldg(xb + (long long)t * V + tok) - __ldg(mb + t)) - logf(__ldg(sb + t)); };

  float* cur = alpha;
  float* nxt = alpha + ns;
  cur[s] = (s == 0 || (s == 1 && L > 0)) ? log_prob(0) : -INFINITY;
  float* ab = nullptr;
  if constexpr (kTrain) {
    ab = alpha_out + b * T * alpha_stride + s;
    if (active) ab[0] = cur[s];
  }
  float lp = (active && n > 1) ? log_prob(1) : 0.f;
  __syncthreads();
  for (int t = 1; t < n; ++t) {
    if (active) {
      const float la1 = cur[s];
      const float la2 = s > 0 ? cur[s - 1] : -INFINITY;
      const float la3 = skip ? cur[s - 2] : -INFINITY;
      float lamax = la1;
      if (la2 > lamax) lamax = la2;
      if (la3 > lamax) lamax = la3;
      if (lamax == -INFINITY) lamax = 0.f;       // cannot do -inf - -inf
      nxt[s] = logf(expf(la1 - lamax) + expf(la2 - lamax) + expf(la3 - lamax)) + lamax + lp;
      if constexpr (kTrain) ab[(long long)t * alpha_stride] = nxt[s];
      if (t + 1 < n) lp = log_prob(t + 1);
    }
    float* tmp = cur;
    cur = nxt;
    nxt = tmp;
    __syncthreads();
  }
  if (s == 0) {
    float nll;
    if (L == 0) {
      nll = -cur[0];
    } else {
      const float l1 = cur[2 * L], l2 = cur[2 * L - 1];
      float m = l1 > l2 ? l1 : l2;
      m = m == -INFINITY ? 0.f : m;
      nll = -(logf(expf(l1 - m) + expf(l2 - m)) + m);
    }
    utt_loss[b] = nll;
  }
}

// ---------------------------------------------------------------------------------------------- gradients
// out[i] = f(p[i]) for the n floats of one row across a warp.  Rows of V floats start on any 4-byte boundary (V =
// 2599), so the 16-byte accesses start at the first aligned element of `out`; `p` must be aligned alike, or the row
// goes one float at a time.
// kRead = false fills the row with f(0) and never touches `p`.
template <bool kRead = true, class F>
__device__ __forceinline__ void warp_row_map(const float* __restrict__ p, float* __restrict__ out, int n, int lane,
                                             F f) {
  int head = (int)(((16 - (reinterpret_cast<uintptr_t>(out) & 15)) & 15) >> 2);
  head = head < n ? head : n;
  auto at = [&](int i) { return kRead ? p[i] : 0.f; };
  if (kRead && (reinterpret_cast<uintptr_t>(p + head) & 15)) {
    for (int i = lane; i < n; i += 32) out[i] = f(at(i));
    return;
  }
  if (lane < head) out[lane] = f(at(lane));
  const int nv = (n - head) >> 2;
  const float4* p4 = reinterpret_cast<const float4*>(p + head);
  float4* o4 = reinterpret_cast<float4*>(out + head);
#pragma unroll 4
  for (int i = lane; i < nv; i += 32) {
    const float4 v = kRead ? __ldg(p4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    o4[i] = make_float4(f(v.x), f(v.y), f(v.z), f(v.w));
  }
  const int done = head + 4 * nv;
  if (done + lane < n) out[done + lane] = f(at(done + lane));
}

// d max_pooling_loss / d logits, one CTA per utterance and one warp per column like max_pool_kernel.  Pass 1 counts
// the positions whose masked, clamped value equals the pooled value (torch's max() / min() backward splits the
// gradient evenly over them; a NaN pooled value ties with the NaNs).  Pass 2 writes every element of the column: the
// share where the position ties, is not masked and lies in the clamp's closed interval [1e-8, 1], zero elsewhere.
__global__ void max_pool_grad_kernel(const float* __restrict__ x, const int32_t* __restrict__ target,
                                     const int32_t* __restrict__ lens, int T, int D, int min_duration,
                                     const float* __restrict__ pooled, const float* __restrict__ upstream,
                                     float* __restrict__ grad) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const long long b = blockIdx.x;
  const int len = lens[b], tgt = target[b];
  const float* xb = x + b * (long long)T * D;
  float* gb = grad + b * (long long)T * D;
  const float g = *upstream, inv_b = __fdiv_rn(1.f, (float)gridDim.x);
  for (int j = warp; j < D; j += nw) {
    const bool kw = j == tgt;
    const float pool = pooled[b * D + j];
    const bool pool_nan = pool != pool;
    // the value the reference pools at frame t, and whether the gradient passes masked_fill and clamp there
    auto pooled_at = [&](int t, float v, bool& passes) {
      const bool masked = t >= len || (kw && t < min_duration);
      const float w = kw ? v : 1.f - v;
      passes = !masked && w >= 1e-8f && w <= 1.f;
      return clamp_nan(masked ? (kw ? 0.f : 1.f) : w, 1e-8f, 1.f);
    };
    int ties = 0;
    for (int t = lane; t < T; t += 32) {
      bool passes;
      const float c = pooled_at(t, xb[(long long)t * D + j], passes);
      ties += pool_nan ? c != c : c == pool;
    }
    for (int o = 16; o > 0; o >>= 1) ties += __shfl_xor_sync(0xffffffffu, ties, o);
    // d(-log(pool)) / B over the ties; 1 - p flips the sign for the other columns
    float share = __fdiv_rn(__fdiv_rn(-inv_b, pool), (float)ties);
    share = __fmul_rn(g, kw ? share : -share);
    for (int t = lane; t < T; t += 32) {
      bool passes;
      const float c = pooled_at(t, xb[(long long)t * D + j], passes);
      const bool tie = pool_nan ? c != c : c == pool;
      gb[(long long)t * D + j] = (tie && passes) ? share : 0.f;
    }
  }
}

// d cross_entropy / d logits, one warp per row: upstream * (softmax - onehot) / count, zeros on an ignored row
__global__ void ce_grad_kernel(const float* __restrict__ x, const int32_t* __restrict__ target, long long B, int C,
                               const float* __restrict__ count, const float* __restrict__ upstream,
                               float* __restrict__ grad) {
  const long long b = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  const float* p = x + b * C;
  float* out = grad + b * C;
  const int t = target[b];
  if (t == kIgnoreIndex) {
    for (int i = lane; i < C; i += 32) out[i] = 0.f;
    return;
  }
  float m, s;
  warp_row_max_sum(p, C, lane, m, s);
  const float g = *upstream, rs = __fdiv_rn(1.f, s), rc = __fdiv_rn(1.f, *count);
  for (int i = lane; i < C; i += 32)
    out[i] = __fmul_rn(g, __fmul_rn(__fmul_rn(expf(p[i] - m), rs) - (i == t ? 1.f : 0.f), rc));
}

// Turns alpha[b][t][s] into the state occupancy gamma = exp(alpha + beta - log p + nll) in place: one CTA per
// utterance, thread s is state s, t walks down in torch's log-space beta recurrence (LossCTC.cpp), beta
// double-buffered in shared memory with one barrier per frame like ctc_alpha_kernel.  Label states that carry the
// same token are merged here, so that ctc_grad_kernel has one writer per token column: the first state of a token
// gets the sum of its occupancies (in label order) and the others -1.  Blank states, and label states whose token is
// the blank, stay as they are (ctc_grad_kernel sums them across a warp).  An infeasible utterance is left alone:
// its rows are NaN whatever alpha holds.
__global__ void ctc_beta_kernel(const float* __restrict__ x, const float* __restrict__ row_max,
                                const float* __restrict__ row_sum, const int32_t* __restrict__ lens,
                                const int32_t* __restrict__ labels, long long label_stride,
                                const int32_t* __restrict__ label_lens, long long T, int V,
                                const float* __restrict__ utt_loss, float* __restrict__ occ, int occ_stride) {
  extern __shared__ float beta[];                // [2][blockDim.x], gamma [2][blockDim.x], next state [blockDim.x]
  const int s = threadIdx.x, ns = blockDim.x;
  float* gam = beta + 2 * ns;
  int* nexts = reinterpret_cast<int*>(gam + 2 * ns);
  const long long b = blockIdx.x;
  const int n = lens[b], L = label_lens[b], S = 2 * L + 1;
  const float nll = utt_loss[b];
  if (n == 0 || nll == INFINITY) return;
  const int32_t* lab = label_of(labels, label_stride, label_lens, b);
  const bool active = s < S;
  const int tok = (active && (s & 1)) ? lab[s >> 1] : 0;
  const bool skip = active && (s & 1) && s + 2 < S && lab[(s >> 1) + 1] != tok;        // l'_{s+2} != l'_s
  // label states of one token: `first` owns the column, `next` is the following state of the same token
  bool first = true;
  int next = -1;
  if (tok != 0) {
    for (int k = 0; k < (s >> 1); ++k) first = first && __ldg(lab + k) != tok;
    for (int k = L - 1; k > (s >> 1); --k)
      if (__ldg(lab + k) == tok) next = 2 * k + 1;
  }
  nexts[s] = next;                               // read after the first frame's barrier
  const float* xb = x + b * T * V;
  const float* mb = row_max + b * T;
  const float* sb = row_sum + b * T;
  float* ob = occ + b * T * occ_stride + s;
  auto log_prob = [&](int t) { return (__ldg(xb + (long long)t * V + tok) - __ldg(mb + t)) - logf(__ldg(sb + t)); };

  float* cur = beta;                             // beta of frame t + 1
  float* nxt = beta + ns;
  float lp = active ? log_prob(n - 1) : 0.f;
  float la = active ? ob[(long long)(n - 1) * occ_stride] : 0.f;
  for (int t = n - 1; t >= 0; --t) {
    float* gt = gam + (t & 1) * ns;
    if (active) {
      float bt;
      if (t == n - 1) {
        bt = (s == 2 * L || s == 2 * L - 1) ? lp : -INFINITY;
      } else {
        const float lb1 = cur[s];
        const float lb2 = s + 1 < S ? cur[s + 1] : -INFINITY;
        const float lb3 = skip ? cur[s + 2] : -INFINITY;
        float lbmax = lb1;
        if (lb2 > lbmax) lbmax = lb2;
        if (lb3 > lbmax) lbmax = lb3;
        if (lbmax == -INFINITY) lbmax = 0.f;
        bt = logf(expf(lb1 - lbmax) + expf(lb2 - lbmax) + expf(lb3 - lbmax)) + lbmax + lp;
      }
      nxt[s] = bt;
      gt[s] = expf(la + bt + nll - lp);
      if (t > 0) {
        lp = log_prob(t - 1);
        la = ob[(long long)(t - 1) * occ_stride];
      }
    }
    float* tmp = cur;
    cur = nxt;
    nxt = tmp;
    __syncthreads();
    // frame t's occupancies are complete; the next frame writes the other half of gam
    if (active) {
      float v = gt[s];
      if (tok != 0) {
        if (first) {
          for (int k = next; k >= 0; k = nexts[k]) v += gt[k];
        } else {
          v = -1.f;
        }
      }
      ob[(long long)t * occ_stride] = v;
    }
  }
}

// d ctc_loss / d logits, one warp per (b, t) row; the hot path, bound by HBM: the logits are read once and the
// gradient is written once.  A frame of a feasible utterance gets upstream * (softmax - occupancy) / B: the warp
// streams the softmax part, then every token column of the label is rewritten by the one state that owns it
// (ctc_beta_kernel merged the states of a token) from the logit read again, and the blank column from the sum of the
// blank occupancies, folded in a fixed order.  Padding rows are zeros; the frames of an infeasible utterance are NaN,
// as torch's backward gives with zero_infinity=False.
__global__ void ctc_grad_kernel(const float* __restrict__ x, const int32_t* __restrict__ lens,
                                const int32_t* __restrict__ labels, long long label_stride,
                                const int32_t* __restrict__ label_lens, long long B, long long T, int V,
                                const float* __restrict__ row_max, const float* __restrict__ row_sum,
                                const float* __restrict__ utt_loss, const float* __restrict__ occ, int occ_stride,
                                const float* __restrict__ upstream, float* __restrict__ grad) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B * T) return;
  const int lane = threadIdx.x & 31;
  const long long b = row / T;
  const float* p = x + row * V;
  float* out = grad + row * V;
  if (row - b * T >= lens[b]) {
    warp_row_map<false>(nullptr, out, V, lane, [](float) { return 0.f; });
    return;
  }
  if (utt_loss[b] == INFINITY) {
    warp_row_map<false>(nullptr, out, V, lane, [](float) { return __int_as_float(0x7fc00000); });
    return;
  }
  const float g = *upstream, m = row_max[row], rs = __fdiv_rn(1.f, row_sum[row]), inv_b = __fdiv_rn(1.f, (float)B);
  auto unit = [&](float v, float gamma) { return __fmul_rn(g, __fmul_rn(__fmul_rn(expf(v - m), rs) - gamma, inv_b)); };
  warp_row_map(p, out, V, lane, [&](float v) { return unit(v, 0.f); });
  __syncwarp();
  const int32_t* lab = label_of(labels, label_stride, label_lens, b);
  const int S = 2 * label_lens[b] + 1;
  const float* ob = occ + row * occ_stride;
  float blank = 0.f;
  for (int s = lane; s < S; s += 32) {
    const float gamma = ob[s];
    const int tok = (s & 1) ? lab[s >> 1] : 0;
    if (tok == 0) blank += gamma;
    else if (!(gamma < 0.f)) out[tok] = unit(p[tok], gamma);
  }
  for (int o = 16; o > 0; o >>= 1) blank += __shfl_xor_sync(0xffffffffu, blank, o);
  if (lane == 0) out[0] = unit(p[0], blank);
}

// Levenshtein distance of the best hypothesis to label b, one warp per utterance: the hypothesis (<= 64 tokens)
// across the lanes (lane l holds columns 2l + 1 and 2l + 2), the label down the rows, so its length is unbounded.
// Row i: E[c] = min(D[i-1][c] + 1, D[i-1][c-1] + (lab != rec)), E[0] = i, and D[i][c] = min_{k <= c} E[k] + c - k,
// a warp prefix-min of E[c] - c.  correct[b] = L_b - distance; best (optional): row b = H, then the hypothesis.
__global__ void ctc_edit_kernel(const int32_t* __restrict__ nhyp, const int32_t* __restrict__ hyp_len,
                                const int32_t* __restrict__ hyp_tokens, int path_beam,
                                const int32_t* __restrict__ labels, long long label_stride,
                                const int32_t* __restrict__ label_lens, long long B, int32_t* __restrict__ correct,
                                int32_t* __restrict__ best) {
  const long long b = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  const int H = nhyp[b] > 0 ? hyp_len[b * path_beam] : 0;
  const int32_t* rec = hyp_tokens + b * path_beam * WEKWS_CTC_MAX_PREFIX;
  const int32_t* lab = label_of(labels, label_stride, label_lens, b);
  const int L = label_lens[b];
  const int c0 = 2 * lane + 1, c1 = 2 * lane + 2;
  const int r0 = c0 <= H ? rec[c0 - 1] : INT32_MIN, r1 = c1 <= H ? rec[c1 - 1] : INT32_MIN;
  if (best) {
    int32_t* o = best + b * (1 + WEKWS_CTC_MAX_PREFIX);
    if (lane == 0) o[0] = H;
    o[c0] = c0 <= H ? r0 : -1;
    o[c1] = c1 <= H ? r1 : -1;
  }
  int d0 = c0, d1 = c1;                          // row 0: D[0][c] = c
  for (int i = 1; i <= L; ++i) {
    const int a = lab[i - 1];
    int left = __shfl_up_sync(0xffffffffu, d1, 1);
    if (lane == 0) left = i - 1;
    const int e0 = min(d0 + 1, left + (a != r0));
    const int e1 = min(d1 + 1, d0 + (a != r1));
    int f = min(e0 - c0, e1 - c1);
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, f, o);
      if (lane >= o) f = min(f, v);
    }
    int before = __shfl_up_sync(0xffffffffu, f, 1);
    before = lane == 0 ? i : min(before, i);
    const int g0 = min(before, e0 - c0), g1 = min(g0, e1 - c1);
    d0 = g0 + c0;
    d1 = g1 + c1;
  }
  const int dist = H == 0 ? L : __shfl_sync(0xffffffffu, (H & 1) ? d0 : d1, (H - 1) >> 1);
  if (lane == 0) correct[b] = L - dist;
}

// loss and accuracy of the batch, in a fixed order:
//   max_pooling: float32 sum of the B*D terms in (i, j) order, / B; acc = correct / B (loss.py:49-87);
//   ce: double sum of the counted terms, as float / count; acc = correct * 100.0 / B (acc_frame);
//   ctc: double sum of the utterance losses, as float / B; acc = (sum of L - distance) * 100.0 / (sum of L) over the
//        non-empty labels (acc_utterance), 0 without validation.
// ce_count (optional, ce): the number of counted rows, which ce_grad_kernel divides by.
__global__ void criterion_reduce_kernel(int kind, long long B, int D, const float* __restrict__ term,
                                        const int32_t* __restrict__ correct, const int32_t* __restrict__ target,
                                        const int32_t* __restrict__ label_lens, int validation,
                                        float* __restrict__ loss, double* __restrict__ acc,
                                        float* __restrict__ ce_count) {
  if (threadIdx.x != 0) return;
  if (kind == kMaxPooling) {
    float sum = 0.f;
    for (long long i = 0; i < B * D; ++i) sum = __fadd_rn(sum, term[i]);
    long long n = 0;
    for (long long b = 0; b < B; ++b) n += correct[b];
    *loss = __fdiv_rn(sum, (float)B);
    *acc = __ddiv_rn((double)n, (double)B);
  } else if (kind == kCe) {
    double sum = 0.0;
    long long counted = 0, n = 0;
    for (long long b = 0; b < B; ++b) {
      if (target[b] != kIgnoreIndex) {
        sum = __dadd_rn(sum, (double)term[b]);
        ++counted;
      }
      n += correct[b];
    }
    *loss = __fdiv_rn((float)sum, (float)counted);
    if (ce_count) *ce_count = (float)counted;
    *acc = __ddiv_rn(__dmul_rn((double)n, 100.0), (double)B);
  } else {
    double sum = 0.0;
    for (long long b = 0; b < B; ++b) sum = __dadd_rn(sum, (double)term[b]);
    *loss = __fdiv_rn((float)sum, (float)B);
    long long words = 0, right = 0;
    if (validation) {
      for (long long b = 0; b < B; ++b) {
        if (label_lens[b] > 0) {
          words += label_lens[b];
          right += correct[b];
        }
      }
    }
    *acc = validation ? __ddiv_rn(__dmul_rn((double)right, 100.0), (double)words) : 0.0;
  }
}

int reduce_launch(int kind, long long B, int D, const float* term, const int32_t* correct, const int32_t* target,
                  const int32_t* label_lens, int validation, float* loss, double* acc, float* ce_count,
                  cudaStream_t st) {
  criterion_reduce_kernel<<<1, 32, 0, st>>>(kind, B, D, term, correct, target, label_lens, validation, loss, acc,
                                            ce_count);
  return check_launch("criterion_reduce_kernel");
}

// caller workspace, carved in 256-byte aligned pieces
struct Carver {
  uint8_t* base;
  size_t off = 0;
  template <class T>
  T* take(long long n) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += ((size_t)n * sizeof(T) + 255) & ~(size_t)255;
    return p;
  }
};

struct CtcWork {
  float *row_max, *row_sum, *utt_loss;
  int32_t *correct, *nhyp, *hyp_len, *hyp_tokens, *node_frame;
  double* hyp_score;
  float* node_prob;
};

size_t ctc_work(Carver& c, long long B, long long T, int validation, CtcWork& w) {
  w.row_max = c.take<float>(B * T);
  w.row_sum = c.take<float>(B * T);
  w.utt_loss = c.take<float>(B);
  if (validation) {
    const long long nh = B * kAccPathBeam;
    w.correct = c.take<int32_t>(B);
    w.nhyp = c.take<int32_t>(B);
    w.hyp_len = c.take<int32_t>(nh);
    w.hyp_score = c.take<double>(nh);
    w.hyp_tokens = c.take<int32_t>(nh * WEKWS_CTC_MAX_PREFIX);
    w.node_frame = c.take<int32_t>(nh * WEKWS_CTC_MAX_PREFIX);
    w.node_prob = c.take<float>(nh * WEKWS_CTC_MAX_PREFIX);
  }
  return c.off;
}

}  // namespace
}  // namespace wekws

using namespace wekws;

extern "C" int64_t wekws_criterion_max_pooling_workspace_bytes(int64_t B, int D) {
  Carver c{nullptr};
  c.take<float>(B * D);
  c.take<int32_t>(B);
  return (int64_t)c.off;
}

// d_pooled != NULL: the training forward
static int max_pooling_forward(const float* d_logits, const int32_t* d_target, const int32_t* d_lens, int64_t B,
                               int64_t T, int D, int min_duration, void* d_workspace, float* d_loss, double* d_acc,
                               float* d_term_loss, int32_t* d_correct, float* d_pooled, cudaStream_t st) {
  WEKWS_REQUIRE(B >= 1 && B < (1ll << 31) && T >= 1 && D >= 1 && D <= 8192,
                "wekws_criterion_max_pooling: bad sizes (B >= 1, T >= 1, 1 <= D <= 8192)");
  WEKWS_REQUIRE(d_logits && d_target && d_lens && d_workspace && d_loss && d_acc,
                "wekws_criterion_max_pooling: null argument");
  Carver c{(uint8_t*)d_workspace};
  float* term = c.take<float>(B * D);
  int32_t* correct = c.take<int32_t>(B);
  if (d_term_loss) term = d_term_loss;
  if (d_correct) correct = d_correct;
  const int nw = D < 8 ? D : 8;
  if (d_pooled)
    max_pool_kernel<true><<<(unsigned)B, nw * 32, (size_t)D * sizeof(float), st>>>(d_logits, d_target, d_lens, (int)T, D,
                                                                                min_duration, term, correct, d_pooled);
  else
    max_pool_kernel<false><<<(unsigned)B, nw * 32, (size_t)D * sizeof(float), st>>>(d_logits, d_target, d_lens, (int)T,
                                                                                 D, min_duration, term, correct, nullptr);
  int rc = check_launch("max_pool_kernel");
  if (rc) return rc;
  return reduce_launch(kMaxPooling, B, D, term, correct, nullptr, nullptr, 0, d_loss, d_acc, nullptr, st);
}

extern "C" int wekws_criterion_max_pooling(const float* d_logits, const int32_t* d_target, const int32_t* d_lens,
                                           int64_t B, int64_t T, int D, int min_duration, void* d_workspace,
                                           float* d_loss, double* d_acc, float* d_term_loss, int32_t* d_correct,
                                           void* stream) {
  return max_pooling_forward(d_logits, d_target, d_lens, B, T, D, min_duration, d_workspace, d_loss, d_acc, d_term_loss,
                             d_correct, nullptr, (cudaStream_t)stream);
}

extern "C" int wekws_criterion_max_pooling_train(const float* d_logits, const int32_t* d_target, const int32_t* d_lens,
                                                 int64_t B, int64_t T, int D, int min_duration, void* d_workspace,
                                                 float* d_loss, double* d_acc, float* d_term_loss, int32_t* d_correct,
                                                 float* d_pooled, void* stream) {
  WEKWS_REQUIRE(d_pooled, "wekws_criterion_max_pooling_train: null argument");
  return max_pooling_forward(d_logits, d_target, d_lens, B, T, D, min_duration, d_workspace, d_loss, d_acc, d_term_loss,
                             d_correct, d_pooled, (cudaStream_t)stream);
}

extern "C" int wekws_criterion_max_pooling_backward(const float* d_logits, const int32_t* d_target,
                                                    const int32_t* d_lens, int64_t B, int64_t T, int D,
                                                    int min_duration, const float* d_pooled, const float* d_upstream,
                                                    float* d_grad, void* stream) {
  WEKWS_REQUIRE(B >= 1 && B < (1ll << 31) && T >= 1 && T < (1ll << 31) && D >= 1 && D <= 8192,
                "wekws_criterion_max_pooling_backward: bad sizes (B >= 1, T >= 1, 1 <= D <= 8192)");
  WEKWS_REQUIRE(d_logits && d_target && d_lens && d_pooled && d_upstream && d_grad,
                "wekws_criterion_max_pooling_backward: null argument");
  const int nw = D < 8 ? D : 8;
  max_pool_grad_kernel<<<(unsigned)B, nw * 32, 0, (cudaStream_t)stream>>>(d_logits, d_target, d_lens, (int)T, D,
                                                                         min_duration, d_pooled, d_upstream, d_grad);
  return check_launch("max_pool_grad_kernel");
}

extern "C" int64_t wekws_criterion_ce_workspace_bytes(int64_t B) {
  Carver c{nullptr};
  c.take<float>(B);
  c.take<int32_t>(B);
  return (int64_t)c.off;
}

static int ce_forward(const float* d_logits, const int32_t* d_target, int64_t B, int C, void* d_workspace, float* d_loss,
                      double* d_acc, float* d_utt_loss, int32_t* d_correct, float* d_count, cudaStream_t st) {
  WEKWS_REQUIRE(B >= 1 && B < (1ll << 31) && C >= 1, "wekws_criterion_ce: bad sizes (B >= 1, C >= 1)");
  WEKWS_REQUIRE(d_logits && d_target && d_workspace && d_loss && d_acc, "wekws_criterion_ce: null argument");
  Carver c{(uint8_t*)d_workspace};
  float* term = c.take<float>(B);
  int32_t* correct = c.take<int32_t>(B);
  if (d_utt_loss) term = d_utt_loss;
  if (d_correct) correct = d_correct;
  const int wpb = 8;
  ce_kernel<<<(unsigned)((B + wpb - 1) / wpb), wpb * 32, 0, st>>>(d_logits, d_target, B, C, term, correct);
  int rc = check_launch("ce_kernel");
  if (rc) return rc;
  return reduce_launch(kCe, B, 1, term, correct, d_target, nullptr, 0, d_loss, d_acc, d_count, st);
}

extern "C" int wekws_criterion_ce(const float* d_logits, const int32_t* d_target, int64_t B, int C, void* d_workspace,
                                  float* d_loss, double* d_acc, float* d_utt_loss, int32_t* d_correct, void* stream) {
  return ce_forward(d_logits, d_target, B, C, d_workspace, d_loss, d_acc, d_utt_loss, d_correct, nullptr,
                    (cudaStream_t)stream);
}

extern "C" int wekws_criterion_ce_train(const float* d_logits, const int32_t* d_target, int64_t B, int C,
                                        void* d_workspace, float* d_loss, double* d_acc, float* d_utt_loss,
                                        int32_t* d_correct, float* d_count, void* stream) {
  WEKWS_REQUIRE(d_count, "wekws_criterion_ce_train: null argument");
  return ce_forward(d_logits, d_target, B, C, d_workspace, d_loss, d_acc, d_utt_loss, d_correct, d_count,
                    (cudaStream_t)stream);
}

extern "C" int wekws_criterion_ce_backward(const float* d_logits, const int32_t* d_target, int64_t B, int C,
                                           const float* d_count, const float* d_upstream, float* d_grad,
                                           void* stream) {
  WEKWS_REQUIRE(B >= 1 && B < (1ll << 31) && C >= 1, "wekws_criterion_ce_backward: bad sizes (B >= 1, C >= 1)");
  WEKWS_REQUIRE(d_logits && d_target && d_count && d_upstream && d_grad, "wekws_criterion_ce_backward: null argument");
  const int wpb = 8;
  ce_grad_kernel<<<(unsigned)((B + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(d_logits, d_target, B, C,
                                                                                       d_count, d_upstream, d_grad);
  return check_launch("ce_grad_kernel");
}

extern "C" int64_t wekws_criterion_ctc_workspace_bytes(int64_t B, int64_t T, int validation) {
  Carver c{nullptr};
  CtcWork w;
  return (int64_t)ctc_work(c, B, T, validation, w);
}

static int ctc_check(const char* who, const float* d_logits, const int32_t* d_lens, int64_t B, int64_t T, int V,
                     const int32_t* d_labels, int64_t label_stride, const int32_t* d_label_lens, int max_label_len) {
  WEKWS_REQUIRE(B >= 1 && B < (1ll << 31) && T >= 1 && T < (1ll << 31) && V >= 1 && V <= 32767,
                "%s: bad sizes (B >= 1, T >= 1, 1 <= V <= 32767)", who);
  WEKWS_REQUIRE(max_label_len >= 0 && max_label_len <= WEKWS_CRITERION_MAX_LABEL && label_stride >= 0,
                "%s: labels of up to %d tokens", who, WEKWS_CRITERION_MAX_LABEL);
  WEKWS_REQUIRE(d_logits && d_lens && d_label_lens && (d_labels || max_label_len == 0), "%s: null argument", who);
  return WEKWS_OK;
}

// d_alpha != NULL: the training forward, which keeps the row normalisers in d_row_max / d_row_sum and alpha
static int ctc_forward(const float* d_logits, const int32_t* d_lens, int64_t B, int64_t T, int V,
                       const int32_t* d_labels, int64_t label_stride, const int32_t* d_label_lens, int max_label_len,
                       int validation, void* d_workspace, float* d_loss, double* d_acc, float* d_utt_loss,
                       int32_t* d_correct, int32_t* d_overflow, int32_t* d_best, float* d_row_max, float* d_row_sum,
                       float* d_alpha, cudaStream_t st) {
  int rc = ctc_check("wekws_criterion_ctc", d_logits, d_lens, B, T, V, d_labels, label_stride, d_label_lens,
                     max_label_len);
  if (rc) return rc;
  WEKWS_REQUIRE(d_workspace && d_loss && d_acc && (d_overflow || !validation), "wekws_criterion_ctc: null argument");
  Carver c{(uint8_t*)d_workspace};
  CtcWork w;
  ctc_work(c, B, T, validation, w);
  if (d_utt_loss) w.utt_loss = d_utt_loss;
  if (d_correct && validation) w.correct = d_correct;
  if (d_alpha) {
    w.row_max = d_row_max;
    w.row_sum = d_row_sum;
  }

  const int wpb = 8;
  const long long rows = B * T;
  ctc_row_kernel<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, st>>>(d_logits, d_lens, B, T, V, w.row_max,
                                                                        w.row_sum);
  if ((rc = check_launch("ctc_row_kernel"))) return rc;
  const int ns = (2 * max_label_len + 1 + 31) / 32 * 32;
  if (d_alpha)
    ctc_alpha_kernel<true><<<(unsigned)B, ns, 2 * ns * sizeof(float), st>>>(
        d_logits, w.row_max, w.row_sum, d_lens, d_labels, label_stride, d_label_lens, T, V, w.utt_loss, d_alpha,
        2 * max_label_len + 1);
  else
    ctc_alpha_kernel<false><<<(unsigned)B, ns, 2 * ns * sizeof(float), st>>>(
        d_logits, w.row_max, w.row_sum, d_lens, d_labels, label_stride, d_label_lens, T, V, w.utt_loss, nullptr, 0);
  if ((rc = check_launch("ctc_alpha_kernel"))) return rc;
  if (validation) {
    CtcArgs a;
    a.probs = d_logits; a.lens = d_lens; a.B = B; a.T = T; a.V = V;
    a.allowed = nullptr; a.n_allowed = 0;
    a.score_beam = kAccScoreBeam < V ? kAccScoreBeam : V; a.path_beam = kAccPathBeam;
    a.frame_offset = 0; a.frame_stride = 1;
    a.state = nullptr; a.reset_state = 1;
    a.nhyp = w.nhyp; a.overflow = d_overflow; a.hyp_len = w.hyp_len; a.hyp_tokens = w.hyp_tokens;
    a.hyp_score = w.hyp_score; a.node_frame = w.node_frame; a.node_prob = w.node_prob;
    a.row_max = w.row_max; a.row_sum = w.row_sum;
    if ((rc = ctc_launch(a, st))) return rc;
    ctc_edit_kernel<<<(unsigned)((B + wpb - 1) / wpb), wpb * 32, 0, st>>>(w.nhyp, w.hyp_len, w.hyp_tokens,
                                                                        kAccPathBeam, d_labels, label_stride,
                                                                        d_label_lens, B, w.correct, d_best);
    if ((rc = check_launch("ctc_edit_kernel"))) return rc;
  }
  return reduce_launch(kCtc, B, 1, w.utt_loss, validation ? w.correct : nullptr, nullptr, d_label_lens, validation,
                       d_loss, d_acc, nullptr, st);
}

extern "C" int wekws_criterion_ctc(const float* d_logits, const int32_t* d_lens, int64_t B, int64_t T, int V,
                                   const int32_t* d_labels, int64_t label_stride, const int32_t* d_label_lens,
                                   int max_label_len, int validation, void* d_workspace, float* d_loss, double* d_acc,
                                   float* d_utt_loss, int32_t* d_correct, int32_t* d_overflow, int32_t* d_best,
                                   void* stream) {
  return ctc_forward(d_logits, d_lens, B, T, V, d_labels, label_stride, d_label_lens, max_label_len, validation,
                     d_workspace, d_loss, d_acc, d_utt_loss, d_correct, d_overflow, d_best, nullptr, nullptr, nullptr,
                     (cudaStream_t)stream);
}

extern "C" int wekws_criterion_ctc_train(const float* d_logits, const int32_t* d_lens, int64_t B, int64_t T, int V,
                                         const int32_t* d_labels, int64_t label_stride, const int32_t* d_label_lens,
                                         int max_label_len, int validation, void* d_workspace, float* d_loss,
                                         double* d_acc, float* d_utt_loss, int32_t* d_correct, int32_t* d_overflow,
                                         int32_t* d_best, float* d_row_max, float* d_row_sum, float* d_alpha,
                                         void* stream) {
  WEKWS_REQUIRE(d_utt_loss && d_row_max && d_row_sum && d_alpha, "wekws_criterion_ctc_train: null argument");
  return ctc_forward(d_logits, d_lens, B, T, V, d_labels, label_stride, d_label_lens, max_label_len, validation,
                     d_workspace, d_loss, d_acc, d_utt_loss, d_correct, d_overflow, d_best, d_row_max, d_row_sum,
                     d_alpha, (cudaStream_t)stream);
}

extern "C" int wekws_criterion_ctc_backward(const float* d_logits, const int32_t* d_lens, int64_t B, int64_t T, int V,
                                            const int32_t* d_labels, int64_t label_stride,
                                            const int32_t* d_label_lens, int max_label_len, const float* d_row_max,
                                            const float* d_row_sum, const float* d_utt_loss, float* d_alpha,
                                            int alpha_is_occupancy, const float* d_upstream, float* d_grad,
                                            void* stream) {
  int rc = ctc_check("wekws_criterion_ctc_backward", d_logits, d_lens, B, T, V, d_labels, label_stride, d_label_lens,
                     max_label_len);
  if (rc) return rc;
  WEKWS_REQUIRE(d_row_max && d_row_sum && d_utt_loss && d_alpha && d_upstream && d_grad,
                "wekws_criterion_ctc_backward: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int stride = 2 * max_label_len + 1;
  if (!alpha_is_occupancy) {
    const int ns = (stride + 31) / 32 * 32;
    ctc_beta_kernel<<<(unsigned)B, ns, 5 * ns * sizeof(float), st>>>(d_logits, d_row_max, d_row_sum, d_lens, d_labels,
                                                                   label_stride, d_label_lens, T, V, d_utt_loss,
                                                                   d_alpha, stride);
    if ((rc = check_launch("ctc_beta_kernel"))) return rc;
  }
  const int wpb = 8;
  const long long rows = B * T;
  ctc_grad_kernel<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, st>>>(d_logits, d_lens, d_labels, label_stride,
                                                                         d_label_lens, B, T, V, d_row_max, d_row_sum,
                                                                         d_utt_loss, d_alpha, stride, d_upstream,
                                                                         d_grad);
  return check_launch("ctc_grad_kernel");
}
