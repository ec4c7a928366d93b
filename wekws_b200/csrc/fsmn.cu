// Fused FSMN forward (SURVEY 8f-4): the whole backbone of wekws/model/fsmn.py:401-495 in one launch --
//   in_linear1 -> in_linear2 -> ReLU -> L x [LinearTransform (no bias) -> FSMNBlock memory -> AffineTransform -> ReLU]
//   -> out_linear1 -> out_linear2 (+ the model's activation), with the 4-D streaming cache (B, proj, pad, L).
// FSMNBlock (fsmn.py:173-253, always built with strides 1,1 -- fsmn.py:384-391): with cat = [cache (pad cols) | p (T)]
//   out[t] = cat[t + lorder - 1] + sum_i wl[i] cat[t + i] + sum_j wr[j] cat[t + lorder + j],   pad = lorder - 1 + rorder
//   new cache = last pad columns of cat.
//
// FP32 FMA path (exact fp32 semantics; the GEMM dims 140 / 250 / 2599 of the shipped fsmn_ctc.yaml are not tensor-core
// shaped).  A CTA owns a tile of S whole streams (S*T <= 64 rows) and walks the network with the activations
// resident in shared memory (two row-major ping-pong buffers); every Linear is a register-tiled GEMM
// (thread = 4 rows x 8 columns, 128 output columns per pass) whose transposed weights [K][Npad] stream from L2 through
// a double-buffered cp.async ring; the last Linear (odim up to thousands) writes straight to global memory.
#include "common.cuh"
#include "fsmn.h"

namespace wekws {

namespace {

constexpr int FN_T = 256;        // threads
constexpr int ROWS = 64;         // tile rows
constexpr int NPASS = 128;       // output columns per GEMM pass
constexpr int KC = 32;           // weight rows per ring chunk
constexpr int RING = KC * NPASS; // floats per ring slot


struct Ring {
  float* buf;      // [2][RING]
  int issued = 0;  // chunks issued / consumed so far (global counters keep the slot parity across GEMMs)
  int used = 0;
};

// issue chunk (k0.., pass np) of W^T [K][Npad] into ring slot (issued & 1)
__device__ __forceinline__ void ring_issue(Ring& r, const float* __restrict__ wt, int K, int Npad, int k0, int np) {
  float* dst = r.buf + (r.issued & 1) * RING;
  const int rows = min(KC, K - k0);
  for (int i = threadIdx.x; i < rows * (NPASS / 4); i += FN_T) {
    const int kk = i / (NPASS / 4), c4 = i - kk * (NPASS / 4);
    cp_async16(dst + kk * NPASS + 4 * c4, wt + (size_t)(k0 + kk) * Npad + np * NPASS + 4 * c4);
  }
  cp_async_commit();
  ++r.issued;
}

// dst[r][n] (or global) = act(src[r][:K] . W[n][:K] + b[n]) for the tile's rows.
//   src: shared, row stride sp (multiple of 4 floats); wt: global W^T [K][Npad], Npad multiple of NPASS; bias: global
//   [Npad] or nullptr.  dst_s != nullptr: shared row stride dp; else global rows via grow[r] (nullptr = skip row).
template <bool RELU>
__device__ void gemm_layer(Ring& ring, const float* __restrict__ src, int sp, int K, const float* __restrict__ wt,
                           const float* __restrict__ bias, int N, int Npad, float* dst_s, int dp, float* const* grow,
                           int gact) {
  const int tid = threadIdx.x;
  const int rg = tid >> 4, cg = tid & 15;           // 16 row groups x 16 column groups
  const int r0 = rg * 4, c0 = cg * 8;
  const int nchunk = (K + KC - 1) / KC, npass = Npad / NPASS;
  ring_issue(ring, wt, K, Npad, 0, 0);
  for (int np = 0; np < npass; ++np) {
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    for (int kc = 0; kc < nchunk; ++kc) {
      cp_async_wait_pending(0);
      __syncthreads();                               // chunk landed; previous chunk's readers are done
      // prefetch the next chunk (of this pass or the first of the next pass) into the other slot
      if (kc + 1 < nchunk) ring_issue(ring, wt, K, Npad, (kc + 1) * KC, np);
      else if (np + 1 < npass) ring_issue(ring, wt, K, Npad, 0, np + 1);
      const float* w = ring.buf + (ring.used & 1) * RING + c0;
      ++ring.used;
      const int k0 = kc * KC, kn = min(KC, K - k0);
      const float* a = src + r0 * sp + k0;
      int k = 0;
      for (; k + 4 <= kn; k += 4) {
        float4 av[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) av[i] = *reinterpret_cast<const float4*>(a + i * sp + k);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float4 w0 = *reinterpret_cast<const float4*>(w + (k + u) * NPASS);
          const float4 w1 = *reinterpret_cast<const float4*>(w + (k + u) * NPASS + 4);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float x = u == 0 ? av[i].x : u == 1 ? av[i].y : u == 2 ? av[i].z : av[i].w;
            acc[i][0] = fmaf(x, w0.x, acc[i][0]); acc[i][1] = fmaf(x, w0.y, acc[i][1]);
            acc[i][2] = fmaf(x, w0.z, acc[i][2]); acc[i][3] = fmaf(x, w0.w, acc[i][3]);
            acc[i][4] = fmaf(x, w1.x, acc[i][4]); acc[i][5] = fmaf(x, w1.y, acc[i][5]);
            acc[i][6] = fmaf(x, w1.z, acc[i][6]); acc[i][7] = fmaf(x, w1.w, acc[i][7]);
          }
        }
      }
      for (; k < kn; ++k) {
        const float4 w0 = *reinterpret_cast<const float4*>(w + k * NPASS);
        const float4 w1 = *reinterpret_cast<const float4*>(w + k * NPASS + 4);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float x = a[i * sp + k];
          acc[i][0] = fmaf(x, w0.x, acc[i][0]); acc[i][1] = fmaf(x, w0.y, acc[i][1]);
          acc[i][2] = fmaf(x, w0.z, acc[i][2]); acc[i][3] = fmaf(x, w0.w, acc[i][3]);
          acc[i][4] = fmaf(x, w1.x, acc[i][4]); acc[i][5] = fmaf(x, w1.y, acc[i][5]);
          acc[i][6] = fmaf(x, w1.z, acc[i][6]); acc[i][7] = fmaf(x, w1.w, acc[i][7]);
        }
      }
    }
    // epilogue of this pass: columns [np*NPASS + c0, +8)
    const int n0 = np * NPASS + c0;
    float b[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) b[j] = bias != nullptr ? __ldg(bias + n0 + j) : 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[j] = acc[i][j] + b[j];
        if (RELU) v[j] = fmaxf(v[j], 0.f);
      }
      if (dst_s != nullptr) {
        if (n0 < dp) {                                // dp >= round-up-8 of N: padding columns hold zeros
          float* d = dst_s + (r0 + i) * dp + n0;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (n0 + j < dp) d[j] = n0 + j < N ? v[j] : 0.f;
        }
      } else {
        float* g = grow[r0 + i];
        if (g != nullptr) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (n0 + j < N) g[n0 + j] = gact == WEKWS_ACT_SIGMOID ? sigmoidf_acc(v[j]) : v[j];
        }
      }
    }
  }
  __syncthreads();                                    // dst complete / ring idle before the caller goes on
}

// training forward: rows [0, rows) of a shared activation buffer (row stride sp, width w) -> saved block `which` of
// layer l, frame (b0 + s) * save_T + save_t0 + t.  Only reads shared memory: the caller's next writer is behind a barrier.
__device__ __forceinline__ void save_rows(const FsmnArgs& a, const float* src, int sp, int w, int which, int l, int b0,
                                          int rows, int T) {
  const long long M = (long long)a.B * a.save_T;
  float* dst = a.saved + fsmn_saved_offset(a, M, which, l);
  for (int idx = threadIdx.x; idx < rows * w; idx += FN_T) {
    const int r = idx / w, c = idx - r * w;
    const int s = r / T, t = r - s * T;
    dst[((long long)(b0 + s) * a.save_T + a.save_t0 + t) * w + c] = src[r * sp + c];
  }
}

// SAVE: the training forward -- the same arithmetic, plus stores of every activation the backward needs
template <bool SAVE>
__device__ __forceinline__ void fsmn_body(const FsmnArgs& a) {
  extern __shared__ __align__(16) float smem[];
  const int T = a.T, S = a.S;
  const int sp0 = a.sp0, sp1 = a.sp1;
  float* buf0 = smem;                         // [ROWS][sp0]: input / linear_dim activations
  float* buf1 = buf0 + ROWS * sp0;            // [ROWS][sp1]: affine / projection activations
  float* mem = buf1 + ROWS * sp1;             // [ROWS][spm]: memory-block output
  const int spm = a.spm;
  Ring ring;
  ring.buf = mem + ROWS * spm;
  __shared__ float* grow[ROWS];
  const int tid = threadIdx.x;
  const int lo = a.lorder, ro = a.rorder, pad = lo - 1 + ro, P = a.proj, L = a.L;

  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    const int b0 = tile * S, Sv = min(S, a.B - b0), rows = Sv * T;
    __syncthreads();                           // previous tile done with shared memory
    // ---- stage the features (+CMVN), zero the padding rows / columns
    for (int idx = tid; idx < ROWS * sp0; idx += FN_T) {
      const int r = idx / sp0, k = idx - r * sp0;
      float v = 0.f;
      if (r < rows && k < a.idim) {
        const int s = r / T, t = r - s * T;
        v = __ldg(a.feats + (size_t)(b0 + s) * a.feat_bstride + (size_t)t * a.idim + k);
        if (a.has_cmvn) v = (v - __ldg(a.w + a.o_mean + k)) * (a.norm_var ? __ldg(a.w + a.o_istd + k) : 1.f);
      }
      buf0[idx] = v;
    }
    if (tid < ROWS) {
      const int s = tid / T, t = tid - s * T;
      grow[tid] = tid < rows ? a.out + (size_t)(b0 + s) * a.out_bstride + (size_t)t * a.odim : nullptr;
    }
    __syncthreads();
    // ---- in_linear1 (no activation), in_linear2 + ReLU                      (fsmn.py:470-472)
    gemm_layer<false>(ring, buf0, sp0, a.idim, a.w + a.o_w_in1, a.w + a.o_b_in1, a.aff_in, a.np_aff_in, buf1, sp1, nullptr, 0);
    if constexpr (SAVE) save_rows(a, buf1, sp1, a.aff_in, 0, 0, b0, rows, T);
    gemm_layer<true>(ring, buf1, sp1, a.aff_in, a.w + a.o_w_in2, a.w + a.o_b_in2, a.lin, a.np_lin, buf0, sp0, nullptr, 0);
    if constexpr (SAVE) save_rows(a, buf0, sp0, a.lin, 1, 0, b0, rows, T);
    // ---- FSMN layers
    for (int l = 0; l < L; ++l) {
      const float* wl = a.w + a.o_layers + (size_t)l * a.layer_stride;
      // LinearTransform (no bias): p = W h                                    (fsmn.py:387)
      gemm_layer<false>(ring, buf0, sp0, a.lin, wl + a.lo_wp, nullptr, P, a.np_proj, buf1, sp1, nullptr, 0);
      if constexpr (SAVE) save_rows(a, buf1, sp1, P, 2, l, b0, rows, T);
      // memory block: taps over cat = [cache | p]; cache read straight from global (fsmn.py:226-248)
      const float* tl = wl + a.lo_taps;        // [lo + ro][P]: left taps then right taps
      for (int idx = tid; idx < rows * P; idx += FN_T) {
        const int r = idx / P, c = idx - r * P;
        const int s = r / T, t = r - s * T;
        const float* cin = a.in_cache ? a.in_cache + (((size_t)(b0 + s) * P + c) * pad) * L + l : nullptr;
        auto cat = [&](int pos) -> float {      // cat[pos], 0 <= pos < pad + T
          if (pos >= pad) return buf1[(s * T + pos - pad) * sp1 + c];
          return cin ? __ldg(cin + (size_t)pos * L) : 0.f;
        };
        float v = cat(t + lo - 1);
        for (int i = 0; i < lo; ++i) v = fmaf(__ldg(tl + i * P + c), cat(t + i), v);
        for (int j = 0; j < ro; ++j) v = fmaf(__ldg(tl + (lo + j) * P + c), cat(t + lo + j), v);
        mem[r * spm + c] = v;
      }
      __syncthreads();                         // every old-cache read of this layer is done (in-place update is legal)
      if constexpr (SAVE) save_rows(a, mem, spm, P, 3, l, b0, rows, T);
      // one thread per (stream, channel) row of the cache, positions ascending: position j takes cat[T + j], which for
      // T < pad is the OLD position T + j > j -- read before it is overwritten, so out_cache may alias in_cache
      for (int sc = tid; sc < Sv * P; sc += FN_T) {
        const int c = sc % P, s = sc / P;
        const size_t g0 = (((size_t)(b0 + s) * P + c) * pad) * L + l;
        for (int j = 0; j < pad; ++j) {
          const int pos = T + j;               // new cache = cat[T .. T + pad)
          float v;
          if (pos >= pad) v = buf1[(s * T + pos - pad) * sp1 + c];
          else v = a.in_cache ? a.in_cache[g0 + (size_t)pos * L] : 0.f;
          a.out_cache[g0 + (size_t)j * L] = v;
        }
      }
      // AffineTransform + ReLU                                               (fsmn.py:389-390)
      gemm_layer<true>(ring, mem, spm, P, wl + a.lo_wa, wl + a.lo_ba, a.lin, a.np_lin, buf0, sp0, nullptr, 0);
      if constexpr (SAVE) save_rows(a, buf0, sp0, a.lin, 4, l, b0, rows, T);
    }
    // ---- out_linear1, out_linear2 (+ activation) -> global                  (fsmn.py:478-479)
    gemm_layer<false>(ring, buf0, sp0, a.lin, a.w + a.o_w_out1, a.w + a.o_b_out1, a.aff_out, a.np_aff_out, buf1, sp1, nullptr, 0);
    if constexpr (SAVE) save_rows(a, buf1, sp1, a.aff_out, 5, 0, b0, rows, T);
    gemm_layer<false>(ring, buf1, sp1, a.aff_out, a.w + a.o_w_out2, a.w + a.o_b_out2, a.odim, a.np_odim, nullptr, 0, grow, a.act);
  }
}

__global__ void __launch_bounds__(FN_T, 1) fsmn_kernel(const FsmnArgs a) { fsmn_body<false>(a); }
__global__ void __launch_bounds__(FN_T, 1) fsmn_train_kernel(const FsmnArgs a) { fsmn_body<true>(a); }

}  // namespace

size_t fsmn_smem_bytes(const FsmnArgs& a) {
  return ((size_t)ROWS * (a.sp0 + a.sp1 + a.spm) + 2 * RING) * sizeof(float);
}
int fsmn_tile_rows() { return ROWS; }
int fsmn_pass_cols() { return NPASS; }

namespace {

template <bool SAVE>
int launch(FsmnArgs a, cudaStream_t st) {
  WEKWS_REQUIRE(a.T >= 1 && a.T <= ROWS && a.B >= 1, "fsmn_launch: chunk of %d frames does not fit a %d-row tile", a.T, ROWS);
  a.S = ROWS / a.T;
  if (a.S > a.B) a.S = a.B;
  a.n_tiles = (a.B + a.S - 1) / a.S;
  const size_t smem = fsmn_smem_bytes(a);
  WEKWS_REQUIRE(smem <= 226 * 1024, "fsmn: layer widths need %zu bytes of shared memory (max 226 KB + static)", smem);
  auto kernel = SAVE ? fsmn_train_kernel : fsmn_kernel;
  if (const int rc = opt_in_smem((const void*)kernel, smem)) return rc;
  const int sms = device_sm_count();
  const int grid = a.n_tiles < sms ? a.n_tiles : sms;
  kernel<<<grid, FN_T, smem, st>>>(a);
  return check_launch(SAVE ? "fsmn_train_kernel" : "fsmn_kernel");
}

}  // namespace

int fsmn_launch(FsmnArgs a, cudaStream_t st) { return launch<false>(a, st); }

int fsmn_train_launch(FsmnArgs a, cudaStream_t st) {
  WEKWS_REQUIRE(a.saved != nullptr && a.save_T >= 1 && a.save_t0 >= 0 && a.save_t0 + a.T <= a.save_T,
                "fsmn_train_launch: bad saved-activation arguments");
  return launch<true>(a, st);
}

}  // namespace wekws
