// CTC prefix beam search + keyword detection on the device (SURVEY 8f-2, CTC models): what the reference does per
// utterance / per frame in pure Python --
//   wekws/model/loss.py:206-312 ctc_prefix_beam_search (whole utterance, wekws/bin/score_ctc.py:198-200) and its
//   streaming twin wekws/bin/stream_kws_ctc.py:124-215 (one frame per call, hypotheses carried), followed by the
//   keyword look-up of score_ctc.py:201-220 / stream_kws_ctc.py:411-434 (is_sublist, sqrt of the product of the
//   token probabilities), and the per-utterance streaming scorer of wekws/bin/stream_score_ctc.py:221-377.
// Bit-exact restatement, including the parts that only exist because of Python object semantics:
//   * probabilities are float32 values promoted to double, every update is the same sequence of double multiplies and
//     adds (no FMA contraction), `math.isclose(p, 0.0, abs_tol=1e-6)` is |p| <= 1e-6;
//   * path nodes are dict OBJECTS shared between hypotheses by the shallow `cur_nodes.copy()`: `nodes[-1]['prob'] = ps`
//     (loss.py:273-275) is visible through every list that holds the same dict.  Nodes therefore live in a pool and the
//     hypotheses hold node ids; "pop + append" (loss.py:296-297) allocates a fresh node;
//   * `next_hyps` is a dict in insertion order and `sorted(..., reverse=True)` is stable: ties keep insertion order;
//   * is_sublist never tests the last possible offset when the prefix is longer than the keyword (score_ctc.py:95).
// One warp per utterance: all lanes scan the frame's V probabilities for the top score_beam entries, lane 0 runs the
// (tiny, inherently sequential) hypothesis update in shared memory.  Utterances are independent -> B warps.
#include <math.h>

#include "common.cuh"
#include "ctc_decode.h"

namespace wekws {
namespace {

constexpr int ML = WEKWS_CTC_MAX_PREFIX;      // longest prefix / node list kept (overflow is flagged)
constexpr int PBM = WEKWS_CTC_MAX_PATH_BEAM;  // path_beam_size limit
constexpr int SBM = WEKWS_CTC_MAX_SCORE_BEAM; // score_beam_size limit
constexpr int NEXTM = PBM * (SBM + 1);        // keys next_hyps can hold: old prefixes + one extension per token
constexpr int POOLM = PBM * ML + PBM * SBM + 8;

struct Hyp {
  double pb, pnb;
  int32_t len, nlen;          // prefix length, node-list length (equal except transiently empty lists)
  int16_t tok[ML];
  int16_t node[ML];
};

struct Work {                 // one utterance's decoder state (shared memory)
  Hyp cur[PBM];
  Hyp next[NEXTM];
  int32_t nframe[POOLM];      // node pool: frame, prob, token
  float nprob[POOLM];
  int16_t ntok[POOLM];
  int16_t remap[POOLM];
  int32_t ncur, npool, overflow;
  uint8_t order[NEXTM];
};

__device__ __forceinline__ bool close0(double p) { return fabs(p) <= 1e-6; }   // math.isclose(p, 0.0, abs_tol=1e-6)

// find the entry with this prefix (tok[0..len) [+ extra]) or insert an empty one -- defaultdict((0.0, 0.0, []))
__device__ int find_or_insert(Work& w, int& nnext, const int16_t* tok, int len, int extra /* -1 = none */) {
  const int L = len + (extra >= 0 ? 1 : 0);
  for (int e = 0; e < nnext; ++e) {
    const Hyp& h = w.next[e];
    if (h.len != L) continue;
    bool same = true;
    for (int i = 0; i < len && same; ++i) same = h.tok[i] == tok[i];
    if (same && extra >= 0) same = h.tok[len] == (int16_t)extra;
    if (same) return e;
  }
  if (nnext >= NEXTM) return -1;
  Hyp& h = w.next[nnext];
  h.pb = 0.0; h.pnb = 0.0; h.len = L; h.nlen = 0;
  for (int i = 0; i < len; ++i) h.tok[i] = tok[i];
  if (extra >= 0) h.tok[len] = (int16_t)extra;
  return nnext++;
}

__device__ __forceinline__ void copy_nodes(Hyp& dst, const Hyp& src) {            // nodes = cur_nodes.copy()
  dst.nlen = src.nlen;
  for (int i = 0; i < src.nlen; ++i) dst.node[i] = src.node[i];
}

__device__ __forceinline__ int new_node(Work& w, int tok, int frame, float prob) {
  if (w.npool >= POOLM) { w.overflow = 1; return POOLM - 1; }
  const int id = w.npool++;
  w.ntok[id] = (int16_t)tok; w.nframe[id] = frame; w.nprob[id] = prob;
  return id;
}

// one frame of loss.py:229-306 / stream_kws_ctc.py:140-213 for the filtered tokens s[0..ns) with probabilities ps[]
__device__ void advance(Work& w, int t, const int* s_idx, const float* s_prob, int ns, int path_beam) {
  int nnext = 0;
  for (int k = 0; k < ns; ++k) {
    const int s = s_idx[k];
    const float psf = s_prob[k];
    const double ps = (double)psf;
    for (int hi = 0; hi < w.ncur; ++hi) {
      const Hyp& c = w.cur[hi];
      const int last = c.len > 0 ? c.tok[c.len - 1] : -1;
      const double pb = c.pb, pnb = c.pnb;
      if (s == 0) {                                               // blank
        const int e = find_or_insert(w, nnext, c.tok, c.len, -1);
        if (e < 0) { w.overflow = 1; continue; }
        Hyp& n = w.next[e];
        n.pb = __dadd_rn(__dadd_rn(n.pb, __dmul_rn(pb, ps)), __dmul_rn(pnb, ps));
        copy_nodes(n, c);
      } else if (s == last) {
        if (!close0(pnb)) {                                       // *ss -> *s
          const int e = find_or_insert(w, nnext, c.tok, c.len, -1);
          if (e < 0) { w.overflow = 1; continue; }
          Hyp& n = w.next[e];
          n.pnb = __dadd_rn(n.pnb, __dmul_rn(pnb, ps));
          copy_nodes(n, c);
          const int id = n.node[n.nlen - 1];
          if (psf > w.nprob[id]) { w.nprob[id] = psf; w.nframe[id] = t; }   // the shared dict is updated in place
        }
        if (!close0(pb)) {                                        // *s-s -> *ss
          if (c.len >= ML) { w.overflow = 1; continue; }
          const int e = find_or_insert(w, nnext, c.tok, c.len, s);
          if (e < 0) { w.overflow = 1; continue; }
          Hyp& n = w.next[e];
          n.pnb = __dadd_rn(n.pnb, __dmul_rn(pb, ps));
          copy_nodes(n, c);
          n.node[n.nlen++] = (int16_t)new_node(w, s, t, psf);
        }
      } else {
        if (c.len >= ML) { w.overflow = 1; continue; }
        const int e = find_or_insert(w, nnext, c.tok, c.len, s);
        if (e < 0) { w.overflow = 1; continue; }
        Hyp& n = w.next[e];
        if (n.nlen > 0) {
          if (psf > w.nprob[n.node[n.nlen - 1]]) n.node[n.nlen - 1] = (int16_t)new_node(w, s, t, psf);   // pop + append
        } else {
          copy_nodes(n, c);
          n.node[n.nlen++] = (int16_t)new_node(w, s, t, psf);
        }
        n.pnb = __dadd_rn(__dadd_rn(n.pnb, __dmul_rn(pb, ps)), __dmul_rn(pnb, ps));
      }
    }
  }
  // stable sort by pb + pnb, descending (insertion sort on an index array keeps ties in insertion order)
  for (int e = 0; e < nnext; ++e) {
    const double key = __dadd_rn(w.next[e].pb, w.next[e].pnb);
    int p = e;
    while (p > 0) {
      const Hyp& o = w.next[w.order[p - 1]];
      if (__dadd_rn(o.pb, o.pnb) >= key) break;
      w.order[p] = w.order[p - 1];
      --p;
    }
    w.order[p] = (uint8_t)e;
  }
  const int keep = nnext < path_beam ? nnext : path_beam;
  // garbage-collect the node pool: keep the nodes the surviving hypotheses reference, ids stay in ascending order
  for (int i = 0; i < w.npool; ++i) w.remap[i] = 0;
  for (int r = 0; r < keep; ++r) {
    const Hyp& h = w.next[w.order[r]];
    for (int i = 0; i < h.nlen; ++i) w.remap[h.node[i]] = 1;
  }
  int live = 0;
  for (int i = 0; i < w.npool; ++i) {
    if (w.remap[i]) {
      w.ntok[live] = w.ntok[i]; w.nframe[live] = w.nframe[i]; w.nprob[live] = w.nprob[i];
      w.remap[i] = (int16_t)live++;
    }
  }
  w.npool = live;
  for (int r = 0; r < keep; ++r) {
    const Hyp& h = w.next[w.order[r]];
    Hyp& d = w.cur[r];
    d.pb = h.pb; d.pnb = h.pnb; d.len = h.len; d.nlen = h.nlen;
    for (int i = 0; i < h.len; ++i) d.tok[i] = h.tok[i];
    for (int i = 0; i < h.nlen; ++i) d.node[i] = w.remap[h.node[i]];
  }
  w.ncur = keep;
}

// keyword-token bitmap over V in shared memory (n_allowed = 0: every token allowed)
__device__ __forceinline__ void build_allow(uint32_t* allow, int V, const int32_t* allowed, int n_allowed, int lane) {
  const int nwords = (V + 31) / 32;
  for (int i = lane; i < nwords; i += 32) allow[i] = n_allowed > 0 ? 0u : 0xffffffffu;
  __syncwarp();
  if (lane == 0) {
    for (int i = 0; i < n_allowed; ++i) {
      const int tkn = allowed[i];
      if (tkn >= 0 && tkn < V) allow[tkn >> 5] |= 1u << (tkn & 31);
    }
  }
}

// the initial hypothesis list [(tuple(), (1.0, 0.0, []))]
__device__ __forceinline__ void reset_hyps(Work& w) {
  w.ncur = 1; w.npool = 0; w.overflow = 0;
  w.cur[0].pb = 1.0; w.cur[0].pnb = 0.0; w.cur[0].len = 0; w.cur[0].nlen = 0;
}

__device__ __forceinline__ void load_hyps(Work& w, const Work* st) {
  w.ncur = st->ncur; w.npool = st->npool; w.overflow = st->overflow;
  for (int h = 0; h < st->ncur; ++h) w.cur[h] = st->cur[h];
  for (int i = 0; i < st->npool; ++i) { w.ntok[i] = st->ntok[i]; w.nframe[i] = st->nframe[i]; w.nprob[i] = st->nprob[i]; }
}

__device__ __forceinline__ void store_hyps(Work* st, const Work& w) {
  st->ncur = w.ncur; st->npool = w.npool; st->overflow = w.overflow;
  for (int h = 0; h < w.ncur; ++h) st->cur[h] = w.cur[h];
  for (int i = 0; i < w.npool; ++i) { st->ntok[i] = w.ntok[i]; st->nframe[i] = w.nframe[i]; st->nprob[i] = w.nprob[i]; }
}

// probs.topk(score_beam) of one frame p[0..V) followed by the prob > 0.05 / keyword-set filter (loss.py:244-255,
// stream_kws_ctc.py:144-161): per-lane candidates, then SB rounds of warp arg-max (ties: lower index first).  Every
// lane returns the same filtered tokens s_idx / s_prob[0..ns) in top-k order.
__device__ __forceinline__ int topk_filter(const float* p, int V, int SB, const uint32_t* allow, int lane, int* s_idx,
                                           float* s_prob) {
  float bv[SBM];
  int bi[SBM];
#pragma unroll
  for (int k = 0; k < SBM; ++k) { bv[k] = -INFINITY; bi[k] = 0x7fffffff; }
  for (int i = lane; i < V; i += 32) {
    const float v = __ldg(p + i);
    if (v > bv[SBM - 1]) {                     // strictly greater: an equal later index never displaces an earlier one
      bv[SBM - 1] = v; bi[SBM - 1] = i;
#pragma unroll
      for (int k = SBM - 1; k > 0; --k) {
        if (bv[k] > bv[k - 1]) {
          const float tv = bv[k]; bv[k] = bv[k - 1]; bv[k - 1] = tv;
          const int ti = bi[k]; bi[k] = bi[k - 1]; bi[k - 1] = ti;
        }
      }
    }
  }
  int ns = 0;
  for (int k = 0; k < SB; ++k) {
    float mv = bv[0];
    int mi = bi[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, mv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
      if (ov > mv || (ov == mv && oi < mi)) { mv = ov; mi = oi; }
    }
    if (bi[0] == mi && mi != 0x7fffffff) {     // the winning lane pops its head
#pragma unroll
      for (int q = 0; q < SBM - 1; ++q) { bv[q] = bv[q + 1]; bi[q] = bi[q + 1]; }
      bv[SBM - 1] = -INFINITY; bi[SBM - 1] = 0x7fffffff;
    }
    // filter: prob > 0.05 (Python float compare of the float32 value) and token in the keyword set
    if (mi != 0x7fffffff && (double)mv > 0.05 && ((allow[mi >> 5] >> (mi & 31)) & 1u)) {
      s_idx[ns] = mi; s_prob[ns] = mv; ++ns;
    }
  }
  return ns;
}

__global__ void __launch_bounds__(32) ctc_prefix_beam_kernel(const CtcArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  Work& w = *reinterpret_cast<Work*>(smem);
  uint32_t* allow = reinterpret_cast<uint32_t*>(smem + sizeof(Work));      // keyword-token bitmap over V (optional)
  const int lane = threadIdx.x;
  const long long b = blockIdx.x;
  const int V = a.V, SB = a.score_beam;
  long long n = a.lens ? (long long)a.lens[b] : a.T;
  n = n < 0 ? 0 : (n > a.T ? a.T : n);

  build_allow(allow, V, a.allowed, a.n_allowed, lane);
  if (lane == 0) {
    // hypotheses: carried state or the initial [(tuple(), (1.0, 0.0, []))]
    Work* st = a.state ? reinterpret_cast<Work*>(a.state + (size_t)b * sizeof(Work)) : nullptr;
    if (st && !a.reset_state) load_hyps(w, st);
    else reset_hyps(w);
  }
  __syncwarp();

  const float* P = a.probs + b * a.T * (long long)V;
  for (long long t = 0; t < n; ++t) {
    int s_idx[SBM];
    float s_prob[SBM];
    const int ns = topk_filter(P + t * V, V, SB, allow, lane, s_idx, s_prob);
    if (ns == 0) continue;                       // loss.py:254-255: the frame is skipped entirely
    if (lane == 0) advance(w, (int)(a.frame_offset + t * a.frame_stride), s_idx, s_prob, ns, a.path_beam);
    __syncwarp();
  }

  if (lane == 0) {
    // hyps = [(prefix, pb + pnb, nodes)]
    a.nhyp[b] = w.ncur;
    a.overflow[b] = w.overflow;
    for (int h = 0; h < a.path_beam; ++h) {
      const long long o = b * a.path_beam + h;
      if (h < w.ncur) {
        const Hyp& c = w.cur[h];
        a.hyp_len[o] = c.len;
        a.hyp_score[o] = __dadd_rn(c.pb, c.pnb);
        for (int i = 0; i < ML; ++i) {
          a.hyp_tokens[o * ML + i] = i < c.len ? c.tok[i] : -1;
          a.node_frame[o * ML + i] = i < c.nlen ? w.nframe[c.node[i]] : -1;
          a.node_prob[o * ML + i] = i < c.nlen ? w.nprob[c.node[i]] : 0.f;
        }
      } else {
        a.hyp_len[o] = -1;
        a.hyp_score[o] = 0.0;
      }
    }
    if (a.state) store_hyps(reinterpret_cast<Work*>(a.state + (size_t)b * sizeof(Work)), w);
  }
}

// score_ctc.py:88-103 (identical copy in stream_kws_ctc.py:105-120), quirk included: for a longer main list the loop
// runs over range(len(main) - len(check)) and never tests the last offset
template <typename Tok>
__device__ int is_sublist(const Tok* main_list, int nm, const int32_t* check, int nc) {
  if (nm < nc) return -1;
  if (nm == nc) {
    for (int i = 0; i < nc; ++i)
      if (main_list[i] != check[i]) return -1;
    return 0;
  }
  for (int i = 0; i < nm - nc; ++i) {
    if (main_list[i] == check[0]) {
      int j = 0;
      while (j < nc && main_list[i + j] == check[j]) ++j;
      if (j == nc) return i;
    }
  }
  return -1;
}

// score_ctc.py:201-220: first hypothesis (in beam order) containing a keyword (in keyword order)
__global__ void ctc_keyword_hit_kernel(const int32_t* __restrict__ nhyp, const int32_t* __restrict__ hyp_len,
                                       const int32_t* __restrict__ hyp_tokens, const int32_t* __restrict__ node_frame,
                                       const float* __restrict__ node_prob, long long B, int path_beam,
                                       const int32_t* __restrict__ kw_tokens, const int32_t* __restrict__ kw_off, int nkw,
                                       int32_t* __restrict__ hit, double* __restrict__ hit_score,
                                       int32_t* __restrict__ start, int32_t* __restrict__ end) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int found = -1, st = 0, en = 0;
  double score = 1.0;
  for (int h = 0; h < nhyp[b] && found < 0; ++h) {
    const long long o = b * path_beam + h;
    const int32_t* pre = hyp_tokens + o * ML;
    for (int k = 0; k < nkw; ++k) {
      const int32_t* lab = kw_tokens + kw_off[k];
      const int nl = kw_off[k + 1] - kw_off[k];
      const int off = is_sublist(pre, hyp_len[o], lab, nl);
      if (off != -1) {
        found = k;
        st = node_frame[o * ML + off];
        en = node_frame[o * ML + off + nl - 1];
        for (int i = off; i < off + nl; ++i) score = __dmul_rn(score, (double)node_prob[o * ML + i]);
        break;
      }
    }
    if (found >= 0) score = sqrt(score);
  }
  hit[b] = found; hit_score[b] = score; start[b] = st; end[b] = en;
}

// ------------------------------------------------------------------------------------------------------------------
// Streaming keyword spotter (stream_kws_ctc.py:400-514, KeyWordSpotter.decode_keywords / execute_detection / the frame
// loop of forward): per frame one beam-search step, then the detection rules on the carried hypotheses.

// execute_detection (stream_kws_ctc.py:411-480) for the current hypotheses: the first one (beam order) containing a
// keyword (dict order); hit_score is multiplied by the token probabilities and square-rooted IN PLACE -- it is only
// ever reset with the hypotheses.  Returns 1 on activation and fills r.
__device__ int detect(const Work& w, const SpotArgs& a, SpotDet& d, wekws_ctc_spot_result& r) {
  int hit = -1, start = 0, end = 0;
  for (int h = 0; h < w.ncur && hit < 0; ++h) {
    const Hyp& c = w.cur[h];
    for (int k = 0; k < a.nkw; ++k) {
      const int32_t* lab = a.kw_tokens + a.kw_off[k];
      const int nl = a.kw_off[k + 1] - a.kw_off[k];
      const int off = is_sublist(c.tok, c.len, lab, nl);
      if (off != -1) {
        hit = k;
        start = w.nframe[c.node[off]];
        end = w.nframe[c.node[off + nl - 1]];
        for (int i = off; i < off + nl; ++i) d.hit_score = __dmul_rn(d.hit_score, (double)w.nprob[c.node[i]]);
        break;
      }
    }
    if (hit >= 0) d.hit_score = sqrt(d.hit_score);
  }
  const int duration = end - start;
  if (hit >= 0 && d.hit_score >= a.threshold && a.min_frames <= duration && duration <= a.max_frames &&
      (d.last_active_pos == -1 || end - d.last_active_pos >= a.interval_frames)) {
    d.last_active_pos = end;
    r.score = d.hit_score; r.state = 1; r.keyword = hit; r.start = start; r.end = end;
    return 1;
  }
  return 0;
}

// KeyWordSpotter.reset(): hypotheses, `activated` and hit_score (the overflow flag of the dropped hypotheses sticks)
__device__ __forceinline__ void reset_detector(Work& w, SpotDet& d) {
  d.overflow |= w.overflow;
  reset_hyps(w);
  d.hit_score = 1.0;
}

// one warp per stream; streams with no frames this call are not touched
__global__ void __launch_bounds__(32) ctc_spot_kernel(const SpotArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  Work& w = *reinterpret_cast<Work*>(smem);
  uint32_t* allow = reinterpret_cast<uint32_t*>(smem + sizeof(Work));
  const int lane = threadIdx.x;
  const long long b = blockIdx.x;
  const int n = a.frames[b];
  if (n <= 0) return;

  build_allow(allow, a.V, a.allowed, a.n_allowed, lane);
  Work* st = reinterpret_cast<Work*>(a.state + (size_t)b * sizeof(Work));
  SpotDet* dp = reinterpret_cast<SpotDet*>(a.det + (size_t)b * sizeof(SpotDet));
  SpotDet d = *dp;                               // lane 0's copy is the one that is used and written back
  if (lane == 0) {
    if (d.live) {
      load_hyps(w, st);
    } else {                                     // reset_all() (stream_kws_ctc.py:521-529) / a new stream
      reset_hyps(w);
      d.hit_score = 1.0; d.total_frames = 0; d.last_active_pos = -1; d.overflow = 0; d.live = 1;
    }
  }
  __syncwarp();

  wekws_ctc_spot_result r;                       // self.result of the last frame processed
  r.score = 0.0; r.state = 0; r.keyword = -1; r.start = 0; r.end = 0; r.overflow = 0; r.reserved = 0;
  const float* P = a.probs + (long long)a.rows[b] * a.V;
  for (int t = 0; t < n; ++t) {
    int s_idx[SBM];
    float s_prob[SBM];
    const int ns = topk_filter(P + (long long)t * a.V, a.V, a.score_beam, allow, lane, s_idx, s_prob);
    int act = 0;
    if (lane == 0) {
      if (ns > 0) advance(w, (int)(d.total_frames + (long long)t * a.frame_stride), s_idx, s_prob, ns, a.path_beam);
      act = detect(w, a, d, r);
      if (act) reset_detector(w, d);             // ... and skip the rest of the chunk (stream_kws_ctc.py:495-501)
    }
    if (__shfl_sync(0xffffffffu, act, 0)) break;
  }

  if (lane == 0) {
    d.total_frames += (long long)n * a.frame_stride;          // every frame of the chunk, even after a break
    // stream_kws_ctc.py:509-512: drop a hypothesis whose first token is more than max_frames old
    if (w.ncur > 0 && w.cur[0].len > 0 && d.total_frames - w.nframe[w.cur[0].node[0]] > a.max_frames)
      reset_detector(w, d);
    d.overflow |= w.overflow;
    store_hyps(st, w);
    *dp = d;
    r.overflow = d.overflow;
    a.result[b] = r;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Streaming scoring of a test set (stream_score_ctc.py:221-377): each utterance decoded frame by frame from the empty
// hypothesis, with that script's own detection rule.

// The detection variables of stream_score_ctc.py:230-234; they live for the whole utterance.
struct ScoreDet {
  double hit_score;
  int32_t hit, start, end;   // hit_keyword (-1 = None), start, end
};

// stream_score_ctc.py:321-347 on a decoded frame.  hit / start / end / hit_score are NOT reset per frame: once a keyword
// has been seen, the loop breaks after the first hypothesis whatever it holds, and hit_score = sqrt(hit_score) runs
// again.  Returns 1 if the (possibly stale) hit activates.
__device__ int stream_detect(const Work& w, const StreamScoreArgs& a, ScoreDet& d) {
  for (int h = 0; h < w.ncur; ++h) {
    const Hyp& c = w.cur[h];
    for (int k = 0; k < a.nkw; ++k) {
      const int32_t* lab = a.kw_tokens + a.kw_off[k];
      const int nl = a.kw_off[k + 1] - a.kw_off[k];
      const int off = is_sublist(c.tok, c.len, lab, nl);
      if (off != -1) {
        d.hit = k;
        d.start = w.nframe[c.node[off]];
        d.end = w.nframe[c.node[off + nl - 1]];
        for (int i = off; i < off + nl; ++i) d.hit_score = __dmul_rn(d.hit_score, (double)w.nprob[c.node[i]]);
        break;
      }
    }
    if (d.hit >= 0) {
      d.hit_score = sqrt(d.hit_score);
      break;
    }
  }
  const int duration = d.end - d.start;
  return d.hit >= 0 && d.hit_score >= a.threshold && a.min_frames <= duration && duration <= a.max_frames;
}

// one warp per utterance, as ctc_prefix_beam_kernel
__global__ void __launch_bounds__(32) ctc_stream_score_kernel(const StreamScoreArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  Work& w = *reinterpret_cast<Work*>(smem);
  uint32_t* allow = reinterpret_cast<uint32_t*>(smem + sizeof(Work));
  const int lane = threadIdx.x;
  const long long b = blockIdx.x;
  long long n = a.lens[b];
  n = n < 0 ? 0 : (n > a.T ? a.T : n);

  build_allow(allow, a.V, a.allowed, a.n_allowed, lane);
  ScoreDet d;                                    // lane 0's copy is the one that is used
  d.hit_score = 1.0; d.hit = -1; d.start = 0; d.end = 0;
  int count = 0, overflow = 0;
  if (lane == 0) reset_hyps(w);
  __syncwarp();

  const float* P = a.probs + b * a.T * (long long)a.V;
  wekws_ctc_stream_detection* out = a.det + b * (long long)a.max_detections;
  for (long long t = 0; t < n; ++t) {
    int s_idx[SBM];
    float s_prob[SBM];
    const int ns = topk_filter(P + t * a.V, a.V, a.score_beam, allow, lane, s_idx, s_prob);
    if (ns == 0) continue;                       // stream_score_ctc.py:260-261: no update and no detection
    if (lane == 0) {
      const int frame = (int)(t * a.frame_stride);
      advance(w, frame, s_idx, s_prob, ns, a.path_beam);
      if (stream_detect(w, a, d)) {
        if (count < a.max_detections) {
          wekws_ctc_stream_detection& r = out[count];
          r.score = d.hit_score; r.keyword = d.hit; r.start = d.start; r.end = d.end; r.frame = frame;
        }
        ++count;
        overflow |= w.overflow;                  // :357-360: hypotheses, hit_keyword and hit_score start over
        reset_hyps(w);
        d.hit = -1; d.hit_score = 1.0;
      }
    }
    __syncwarp();
  }

  if (lane == 0) {
    a.count[b] = count;
    a.overflow[b] = overflow | w.overflow;
  }
}

// the dynamic shared-memory opt-in of a kernel, once per device and size
int opt_in_smem(const void* kern, size_t smem, size_t* attr_bytes /* [64] */) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && attr_bytes[dev] < smem) {
    WEKWS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_bytes[dev] = smem;
  }
  return WEKWS_OK;
}

}  // namespace

size_t ctc_state_bytes() { return sizeof(Work); }
size_t ctc_spot_state_bytes() { return sizeof(SpotDet); }

int ctc_launch(const CtcArgs& a, cudaStream_t st) {
  const size_t smem = sizeof(Work) + (size_t)((a.V + 31) / 32) * 4;
  WEKWS_REQUIRE(smem <= 227 * 1024, "ctc decode: vocabulary %d too large for the shared-memory token bitmap", a.V);
  static size_t attr_bytes[64] = {0};                  // per device: the largest dynamic size opted into so far
  const int rc = opt_in_smem((const void*)ctc_prefix_beam_kernel, smem, attr_bytes);
  if (rc != WEKWS_OK) return rc;
  ctc_prefix_beam_kernel<<<(unsigned)a.B, 32, smem, st>>>(a);
  return check_launch("ctc_prefix_beam_kernel");
}

int ctc_spot_launch(const SpotArgs& a, cudaStream_t st) {
  const size_t smem = sizeof(Work) + (size_t)((a.V + 31) / 32) * 4;
  WEKWS_REQUIRE(smem <= 227 * 1024, "ctc spot: vocabulary %d too large for the shared-memory token bitmap", a.V);
  static size_t attr_bytes[64] = {0};
  const int rc = opt_in_smem((const void*)ctc_spot_kernel, smem, attr_bytes);
  if (rc != WEKWS_OK) return rc;
  ctc_spot_kernel<<<(unsigned)a.B, 32, smem, st>>>(a);
  return check_launch("ctc_spot_kernel");
}

int ctc_stream_score_launch(const StreamScoreArgs& a, cudaStream_t st) {
  const size_t smem = sizeof(Work) + (size_t)((a.V + 31) / 32) * 4;
  WEKWS_REQUIRE(smem <= 227 * 1024, "ctc stream score: vocabulary %d too large for the shared-memory token bitmap", a.V);
  static size_t attr_bytes[64] = {0};
  const int rc = opt_in_smem((const void*)ctc_stream_score_kernel, smem, attr_bytes);
  if (rc != WEKWS_OK) return rc;
  ctc_stream_score_kernel<<<(unsigned)a.B, 32, smem, st>>>(a);
  return check_launch("ctc_stream_score_kernel");
}

int ctc_hit_launch(const int32_t* nhyp, const int32_t* hyp_len, const int32_t* hyp_tokens, const int32_t* node_frame,
                   const float* node_prob, long long B, int path_beam, const int32_t* kw_tokens, const int32_t* kw_off,
                   int nkw, int32_t* hit, double* hit_score, int32_t* start, int32_t* end, cudaStream_t st) {
  const int nt = 64;
  ctc_keyword_hit_kernel<<<(unsigned)((B + nt - 1) / nt), nt, 0, st>>>(nhyp, hyp_len, hyp_tokens, node_frame, node_prob, B,
                                                                     path_beam, kw_tokens, kw_off, nkw, hit, hit_score,
                                                                     start, end);
  return check_launch("ctc_keyword_hit_kernel");
}

}  // namespace wekws

using namespace wekws;

extern "C" int64_t wekws_ctc_state_bytes(void) { return (int64_t)ctc_state_bytes(); }

extern "C" int wekws_ctc_prefix_beam_search(const float* d_probs, const int32_t* d_lens, int64_t B, int64_t T, int V,
                                            const int32_t* d_keyword_tokens, int n_keyword_tokens, int score_beam_size,
                                            int path_beam_size, int64_t frame_offset, int frame_stride, void* d_state,
                                            int reset_state, int32_t* d_nhyp, int32_t* d_hyp_len, int32_t* d_hyp_tokens,
                                            double* d_hyp_score, int32_t* d_node_frame, float* d_node_prob,
                                            int32_t* d_overflow, void* stream) {
  WEKWS_REQUIRE(B >= 0 && T >= 0 && V >= 1 && V <= 32767, "wekws_ctc_prefix_beam_search: bad sizes (vocabulary <= 32767)");
  WEKWS_REQUIRE(score_beam_size >= 1 && score_beam_size <= WEKWS_CTC_MAX_SCORE_BEAM && score_beam_size <= V,
                "score_beam_size %d out of range (1..%d)", score_beam_size, WEKWS_CTC_MAX_SCORE_BEAM);
  WEKWS_REQUIRE(path_beam_size >= 1 && path_beam_size <= WEKWS_CTC_MAX_PATH_BEAM, "path_beam_size %d out of range (1..%d)",
                path_beam_size, WEKWS_CTC_MAX_PATH_BEAM);
  WEKWS_REQUIRE(n_keyword_tokens >= 0 && (n_keyword_tokens == 0 || d_keyword_tokens), "keyword token set is null");
  WEKWS_REQUIRE(frame_stride >= 1, "frame_stride must be >= 1");
  if (B == 0) return WEKWS_OK;
  WEKWS_REQUIRE((d_probs || T == 0) && d_nhyp && d_hyp_len && d_hyp_tokens && d_hyp_score && d_node_frame && d_node_prob &&
                    d_overflow,
                "wekws_ctc_prefix_beam_search: null argument");
  CtcArgs a;
  a.probs = d_probs; a.lens = d_lens; a.B = B; a.T = T; a.V = V;
  a.allowed = d_keyword_tokens; a.n_allowed = n_keyword_tokens;
  a.score_beam = score_beam_size; a.path_beam = path_beam_size;
  a.frame_offset = frame_offset; a.frame_stride = frame_stride;
  a.state = (uint8_t*)d_state; a.reset_state = reset_state;
  a.nhyp = d_nhyp; a.overflow = d_overflow; a.hyp_len = d_hyp_len; a.hyp_tokens = d_hyp_tokens; a.hyp_score = d_hyp_score;
  a.node_frame = d_node_frame; a.node_prob = d_node_prob;
  return ctc_launch(a, (cudaStream_t)stream);
}

extern "C" int wekws_ctc_keyword_hit(const int32_t* d_nhyp, const int32_t* d_hyp_len, const int32_t* d_hyp_tokens,
                                     const int32_t* d_node_frame, const float* d_node_prob, int64_t B, int path_beam_size,
                                     const int32_t* d_kw_tokens, const int32_t* d_kw_offsets, int num_keywords,
                                     int32_t* d_hit, double* d_hit_score, int32_t* d_start, int32_t* d_end, void* stream) {
  WEKWS_REQUIRE(B >= 0 && path_beam_size >= 1 && num_keywords >= 1, "wekws_ctc_keyword_hit: bad sizes");
  if (B == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_nhyp && d_hyp_len && d_hyp_tokens && d_node_frame && d_node_prob && d_kw_tokens && d_kw_offsets && d_hit &&
                    d_hit_score && d_start && d_end,
                "wekws_ctc_keyword_hit: null argument");
  return ctc_hit_launch(d_nhyp, d_hyp_len, d_hyp_tokens, d_node_frame, d_node_prob, B, path_beam_size, d_kw_tokens,
                        d_kw_offsets, num_keywords, d_hit, d_hit_score, d_start, d_end, (cudaStream_t)stream);
}

extern "C" int64_t wekws_ctc_spot_state_bytes(void) { return (int64_t)ctc_spot_state_bytes(); }

extern "C" int wekws_ctc_spot(const float* d_probs, int V, const int32_t* d_rows, const int32_t* d_frames, int64_t B,
                              const int32_t* d_keyword_tokens, int n_keyword_tokens, const int32_t* d_kw_tokens,
                              const int32_t* d_kw_offsets, int num_keywords, int score_beam_size, int path_beam_size,
                              int frame_stride, double threshold, int min_frames, int max_frames, int interval_frames,
                              void* d_state, void* d_det, wekws_ctc_spot_result* d_result, void* stream) {
  WEKWS_REQUIRE(B >= 0 && B < (1ll << 31) && V >= 1 && V <= 32767, "wekws_ctc_spot: bad sizes (vocabulary <= 32767)");
  WEKWS_REQUIRE(score_beam_size >= 1 && score_beam_size <= WEKWS_CTC_MAX_SCORE_BEAM && score_beam_size <= V,
                "score_beam_size %d out of range (1..%d)", score_beam_size, WEKWS_CTC_MAX_SCORE_BEAM);
  WEKWS_REQUIRE(path_beam_size >= 1 && path_beam_size <= WEKWS_CTC_MAX_PATH_BEAM, "path_beam_size %d out of range (1..%d)",
                path_beam_size, WEKWS_CTC_MAX_PATH_BEAM);
  WEKWS_REQUIRE(n_keyword_tokens >= 0 && (n_keyword_tokens == 0 || d_keyword_tokens), "keyword token set is null");
  WEKWS_REQUIRE(num_keywords >= 1 && d_kw_tokens && d_kw_offsets, "wekws_ctc_spot: no keywords");
  WEKWS_REQUIRE(frame_stride >= 1, "frame_stride must be >= 1");
  if (B == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_probs && d_rows && d_frames && d_state && d_det && d_result, "wekws_ctc_spot: null argument");
  SpotArgs a;
  a.probs = d_probs; a.rows = d_rows; a.frames = d_frames; a.B = B; a.V = V;
  a.allowed = d_keyword_tokens; a.n_allowed = n_keyword_tokens;
  a.kw_tokens = d_kw_tokens; a.kw_off = d_kw_offsets; a.nkw = num_keywords;
  a.score_beam = score_beam_size; a.path_beam = path_beam_size; a.frame_stride = frame_stride;
  a.threshold = threshold; a.min_frames = min_frames; a.max_frames = max_frames; a.interval_frames = interval_frames;
  a.state = (uint8_t*)d_state; a.det = (uint8_t*)d_det; a.result = d_result;
  return ctc_spot_launch(a, (cudaStream_t)stream);
}

static_assert(sizeof(wekws_ctc_stream_detection) == 24, "wekws_ctc_stream_detection layout is part of the C ABI");

extern "C" int wekws_ctc_stream_score(const float* d_probs, const int32_t* d_lens, int64_t B, int64_t T, int V,
                                      const int32_t* d_keyword_tokens, int n_keyword_tokens, const int32_t* d_kw_tokens,
                                      const int32_t* d_kw_offsets, int num_keywords, int score_beam_size,
                                      int path_beam_size, int frame_stride, double threshold, int min_frames,
                                      int max_frames, int max_detections, int32_t* d_count,
                                      wekws_ctc_stream_detection* d_detections, int32_t* d_overflow, void* stream) {
  WEKWS_REQUIRE(B >= 0 && B < (1ll << 31) && T >= 0 && V >= 1 && V <= 32767,
                "wekws_ctc_stream_score: bad sizes (vocabulary <= 32767)");
  WEKWS_REQUIRE(T * (int64_t)frame_stride <= INT32_MAX, "wekws_ctc_stream_score: frame numbers overflow int32");
  WEKWS_REQUIRE(score_beam_size >= 1 && score_beam_size <= WEKWS_CTC_MAX_SCORE_BEAM && score_beam_size <= V,
                "score_beam_size %d out of range (1..%d)", score_beam_size, WEKWS_CTC_MAX_SCORE_BEAM);
  WEKWS_REQUIRE(path_beam_size >= 1 && path_beam_size <= WEKWS_CTC_MAX_PATH_BEAM, "path_beam_size %d out of range (1..%d)",
                path_beam_size, WEKWS_CTC_MAX_PATH_BEAM);
  WEKWS_REQUIRE(n_keyword_tokens >= 0 && (n_keyword_tokens == 0 || d_keyword_tokens), "keyword token set is null");
  WEKWS_REQUIRE(num_keywords >= 1 && d_kw_tokens && d_kw_offsets, "wekws_ctc_stream_score: no keywords");
  WEKWS_REQUIRE(frame_stride >= 1, "frame_stride must be >= 1");
  WEKWS_REQUIRE(max_detections >= 0, "max_detections must be >= 0");
  if (B == 0) return WEKWS_OK;
  WEKWS_REQUIRE((d_probs || T == 0) && d_lens && d_count && d_overflow && (d_detections || max_detections == 0),
                "wekws_ctc_stream_score: null argument");
  StreamScoreArgs a;
  a.probs = d_probs; a.lens = d_lens; a.B = B; a.T = T; a.V = V;
  a.allowed = d_keyword_tokens; a.n_allowed = n_keyword_tokens;
  a.kw_tokens = d_kw_tokens; a.kw_off = d_kw_offsets; a.nkw = num_keywords;
  a.score_beam = score_beam_size; a.path_beam = path_beam_size; a.frame_stride = frame_stride;
  a.threshold = threshold; a.min_frames = min_frames; a.max_frames = max_frames;
  a.max_detections = max_detections; a.count = d_count; a.det = d_detections; a.overflow = d_overflow;
  return ctc_stream_score_launch(a, (cudaStream_t)stream);
}
