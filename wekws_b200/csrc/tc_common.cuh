// sm_90a building blocks for the tensor-core path: mbarrier, bulk async copies (TMA engine), warpgroup MMA
// (wgmma) with shared-memory descriptors, and the bf16 "x3" operand split (x ~ b0 + b1, products b0*w0 + b1*w0 +
// b0*w1, ~2^-17 relative error).
//
// Operand layout used everywhere here: K-major, SWIZZLE_128B, bf16.  A row of a 64-wide K slab
// is 128 bytes = 8 chunks of 16 B; chunk j of row r lives at position j ^ (r & 7); rows are
// packed 8 x 128 B = 1024 B per core-matrix group (SBO = 1024), so an [R][64] bf16 operand is a
// dense R*128-byte image whose base must be 1024-byte aligned.  One wgmma consumes K = 16
// (32 bytes of every row): the K step advances the descriptor start address by 32 bytes.
//
// wgmma register fragments (m64nNk16, warp w = 0..3 of the warpgroup, lane l): the accumulator element d[4 j + 2 h + e]
// is row 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e; the A operand from registers is four packed bf16 pairs
// {(r, k), (r + 8, k), (r, k + 8), (r + 8, k + 8)} with r = 16 w + l / 4, k = 2 (l % 4) (+1 in the high half).  An
// accumulator of columns [16 s, 16 s + 16) is therefore exactly the A fragment of K step s of a following GEMM.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace wekws {
namespace tc {

// ------------------------------------------------------------------- host: pre-swizzled weight images
// round-to-nearest-even fp32 -> bf16 (as __floats2bfloat162_rn does on the device)
inline uint16_t bf16_rn(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  if ((u & 0x7F800000u) == 0x7F800000u) return (uint16_t)(u >> 16);      // inf / nan
  u += 0x7FFFu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
inline float bf16_to_f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
// The hi and lo images of one `rows` x 64 K slab of a weight matrix in the layout above: element (n, k) of the slab is
// w[n * n_stride + k * k_stride], split as hi = bf16(w), lo = bf16(w - hi).  hi goes to dst, lo to dst + rows * 128;
// rows n >= n_valid and columns k >= k_valid are zero.
inline void write_sw128_bf16x3(uint8_t* dst, int rows, const float* w, ptrdiff_t n_stride, ptrdiff_t k_stride,
                               int n_valid, int k_valid) {
  uint8_t* lo_img = dst + (size_t)rows * 128;
  memset(dst, 0, (size_t)rows * 256);
  for (int n = 0; n < rows && n < n_valid; ++n)
    for (int kk = 0; kk < 64 && kk < k_valid; ++kk) {
      const float v = w[n * n_stride + kk * k_stride];
      const uint16_t hi = bf16_rn(v), lo = bf16_rn(v - bf16_to_f(hi));
      const size_t off = (size_t)n * 128 + (size_t)(((kk >> 3) ^ (n & 7)) << 4) + (size_t)(kk & 7) * 2;
      memcpy(dst + off, &hi, 2);
      memcpy(lo_img + off, &lo, 2);
    }
}

// ------------------------------------------------------------------------------ device
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
#ifdef WEKWS_MBAR_WATCHDOG
// debug build: a wait that never completes reports which barrier it was (plus every warp's last progress mark)
// and traps instead of hanging the GPU
static __device__ int wd_marks[256][20];
__device__ __forceinline__ void wd_mark(int v) {
  if ((threadIdx.x & 31) == 0) *(volatile int*)&wd_marks[blockIdx.x & 255][(threadIdx.x >> 5) % 20] = v;
}
static __device__ __noinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (long long spin = 0; spin < (1ll << 22); ++spin) {
    uint32_t done;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
  }
  if ((threadIdx.x & 31) == 0 && blockIdx.x == 0) {
    volatile int* m = wd_marks[0];
    printf("mbar_wait timeout: thread %d barrier@smem 0x%x parity %u marks c0 %d c1 %d c2 %d c3 %d c4 %d c8 %d c12 %d c15 %d iss %d ld0 %d ld1 %d\n",
           (int)threadIdx.x, smem_u32(bar), parity, m[0], m[1], m[2], m[3], m[4], m[8], m[12], m[15], m[16], m[17], m[18]);
  }
  for (int i = 0; i < 2000; ++i) __nanosleep(100000);       // let the other waiters report too
  __trap();
}
#else
__device__ __forceinline__ void wd_mark(int) {}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
#endif

// same, for single-lane service warps: back off between polls so the spin does not eat issue slots
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
#ifdef WEKWS_MBAR_WATCHDOG
  mbar_wait(bar, parity);
  return;
#endif
  uint32_t done = 0;
  while (true) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) break;
    __nanosleep(40);
  }
}

// -------------------------------------------------------------------- bulk async copies
// global -> shared, completion signalled on an mbarrier as transaction bytes (16 B granularity)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// generic-proxy writes (st.shared) -> visible to the async proxy (wgmma / bulk copies)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// --------------------------------------------------------------------------------- wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Hopper register reallocation between the warpgroups of a CTA (warpgroup-collective): dec gives registers back to the
// CTA's pool, inc waits until the pool can raise this warpgroup to N registers per thread
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
// keeps the compiler from moving accesses of an accumulator across the asynchronous MMAs that own it
template <int R>
__device__ __forceinline__ void wgmma_reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D (+)= A * B^T, bf16 x bf16 -> fp32, issued by a whole warpgroup; B is an [N][K] K-major SW128 image in shared
// memory; A either four registers (_rs) or an [64][K] K-major SW128 image (_ss).  accumulate == 0 overwrites D.
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(desc_b), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// ------------------------------------------------------------------- packed f32x2 math (FFMA2)
// Two fp32 values in one 64-bit register (lo = first); element-wise fp32 math on the pair.
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pack2(float lo, float hi) {
  f32x2 d;
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(lo), "f"(hi));
  return d;
}
__device__ __forceinline__ void unpack2(f32x2 v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
  return pack2(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}
// 16-byte shared-memory accesses as two packed pairs (shared-window addresses)
__device__ __forceinline__ void lds_2x2(uint32_t addr, f32x2& a, f32x2& b) {
  asm volatile("ld.shared.v2.b64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "r"(addr));
}
__device__ __forceinline__ void sts_2x2(uint32_t addr, f32x2 a, f32x2 b) {
  asm volatile("st.shared.v2.b64 [%0], {%1, %2};" ::"r"(addr), "l"(a), "l"(b) : "memory");
}

// bf16 split of a packed pair: hi = bf16x2(x), its two values back as fp32, the exact residual r = x - hi,
// lo = bf16x2(r).
//   split_pair_rn      : hi rounded to nearest (|r| <= 2^-9 |x|), no activation
//   split_pair_rz_relu : y = max(x, 0) folded in: hi = RZ(relu(x)) via cvt.rz.relu, so r = x - hi keeps the sign of x
//                        (r >= 0 for x >= 0, r = x < 0 for x < 0) and lo = RN(relu(r)) -- no separate max
__device__ __forceinline__ void split_pair_rn(f32x2 x, uint32_t& hi, uint32_t& lo) {
  float x0, x1, r0, r1;
  unpack2(x, x0, x1);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
  const f32x2 hf = pack2(__uint_as_float(hi << 16), __uint_as_float(hi & 0xffff0000u));
  const f32x2 neg1 = 0xbf800000bf800000ull;                   // {-1.0f, -1.0f}
  unpack2(fma2(hf, neg1, x), r0, r1);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(r1), "f"(r0));
}
__device__ __forceinline__ void split_pair_rz_relu(f32x2 x, uint32_t& hi, uint32_t& lo) {
  float x0, x1, r0, r1;
  unpack2(x, x0, x1);
  asm("cvt.rz.relu.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
  const f32x2 hf = pack2(__uint_as_float(hi << 16), __uint_as_float(hi & 0xffff0000u));
  const f32x2 neg1 = 0xbf800000bf800000ull;
  unpack2(fma2(hf, neg1, x), r0, r1);
  asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(r1), "f"(r0));
}

// wgmma shared-memory descriptor, K-major SWIZZLE_128B (PTX ISA "Matrix Descriptor Format", sm_90)
__device__ __forceinline__ uint64_t make_sdesc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);          // start address, 16-byte units   [0,14)
  d |= (uint64_t)1 << 16;                                // leading byte offset (unused)   [16,30)
  d |= (uint64_t)(1024 >> 4) << 32;                      // stride byte offset = 1024 B    [32,46)
  d |= (uint64_t)1 << 62;                                // layout type SWIZZLE_128B       [62,64)
  return d;
}

// byte offset of the 16-byte chunk `chunk` (0..7) of row `row` inside a K-major SW128 operand image
__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk) {
  return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4));
}

// ------------------------------------------------------------------------- bf16 x3 split
// x ~ b0 + b1 with b0 = bf16(x), b1 = bf16(x - b0); two values packed per 32-bit word (lo = first)
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
  const float r0 = x0 - __low2float(h), r1 = x1 - __high2float(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(r0, r1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// splits 8 consecutive K values and stores them as one 16-byte chunk into each operand image
__device__ __forceinline__ void split_store8(const float (&v)[8], uint8_t* img_hi, uint8_t* img_lo, uint32_t off) {
  uint4 h, l;
  split2(v[0], v[1], h.x, l.x);
  split2(v[2], v[3], h.y, l.y);
  split2(v[4], v[5], h.z, l.z);
  split2(v[6], v[7], h.w, l.w);
  *reinterpret_cast<uint4*>(img_hi + off) = h;
  *reinterpret_cast<uint4*>(img_lo + off) = l;
}

}  // namespace tc
}  // namespace wekws
