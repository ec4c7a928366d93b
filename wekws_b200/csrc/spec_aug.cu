// SpecAugment of the training front-end (wekws/dataset/processor.py spec_aug): zeros in the masked frames and feature
// columns of each utterance's valid frames.  The host draws the masks with Python's `random` in the reference's order
// and sends the table up; this kernel only stores zeros, so every other element is neither read nor rewritten.
#include "common.cuh"

namespace wekws {
namespace {

// masks of row b: num_t (start, end) frame ranges, then num_f (start, end) column ranges, ends exclusive
__global__ void spec_aug_kernel(float* __restrict__ feats, const int32_t* __restrict__ frames,
                                const int32_t* __restrict__ masks, long long B, long long T, int D, int num_t,
                                int num_f) {
  const long long rows = B * T;
  const int nm = 2 * (num_t + num_f);
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const long long b = r / T, t = r % T;
    if (t >= __ldg(frames + b)) continue;                       // block-uniform
    const int32_t* mk = masks + b * nm;
    bool row_masked = false;
    for (int i = 0; i < num_t; ++i) row_masked |= t >= __ldg(mk + 2 * i) && t < __ldg(mk + 2 * i + 1);
    float* row = feats + r * D;
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      bool z = row_masked;
      for (int i = num_t; i < num_t + num_f; ++i) z |= d >= __ldg(mk + 2 * i) && d < __ldg(mk + 2 * i + 1);
      if (z) row[d] = 0.f;
    }
  }
}

}  // namespace
}  // namespace wekws

using namespace wekws;

extern "C" int wekws_spec_aug(float* d_feats, const int32_t* d_frames, int64_t B, int64_t T, int D,
                              const int32_t* d_masks, int num_t_mask, int num_f_mask, void* stream) {
  WEKWS_REQUIRE(B >= 0 && T >= 0 && D >= 0 && num_t_mask >= 0 && num_f_mask >= 0, "wekws_spec_aug: negative size");
  if (B == 0 || T == 0 || D == 0 || num_t_mask + num_f_mask == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_feats && d_frames && d_masks, "wekws_spec_aug: null pointer");
  const long long rows = B * T;
  const int grid = (int)(rows < (1 << 20) ? rows : (1 << 20));
  const int threads = D <= 64 ? 64 : 128;
  spec_aug_kernel<<<grid, threads, 0, (cudaStream_t)stream>>>(d_feats, d_frames, d_masks, B, T, D, num_t_mask,
                                                              num_f_mask);
  return check_launch("spec_aug_kernel");
}
