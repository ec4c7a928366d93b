// Host side of the model C-ABI: tensor registry keyed by the reference's state_dict names,
// eval-mode BatchNorm folding, weight packing for the fused kernels, forward dispatch.
//
// Folding (SURVEY.md 8a "Folded per-block math"; mdtc.py:55-59,115-118; tcn.py:75-84,101-114):
// for each BatchNorm with s = gamma / sqrt(var + 1e-5), t = beta - mean * s,
//     BN(conv(x; W, b)) = conv(x; W * s[out], b * s + t)
// computed in double and rounded once to fp32.
#include <math.h>
#include <stdarg.h>
#include <string.h>

#include <map>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "conv_backbone.h"
#include "gru.h"
#include "gru_tc.h"
#include "mdtc_tc.h"
#include "tcn_tc.h"
#include "dstcn_tc.h"
#include "fsmn.h"
#include "mdtc_head_train.h"
#include "mdtc_train.h"
#include "tcn_train.h"
#include "linear_tc.h"
#include "cls_head.h"
#include "tc_common.cuh"

namespace wekws {

static thread_local std::string tl_error;
std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  tl_error = buf;
}

int device_sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

// cudaFuncAttributeMaxDynamicSharedMemorySize belongs to the kernel function on a device, not to a caller: every
// caller in the process shares it.  So it is only ever raised, per device and kernel instance, to the largest size any
// launch has needed; a later, smaller launch never lowers it under a concurrent larger one.  The starting limit is
// read from the kernel, not assumed: without an opt-in, static and dynamic shared memory share 48 KB.
int opt_in_smem(const void* kernel, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> limit;   // (device, kernel) -> its dynamic shared-memory limit
  int dev = 0;
  WEKWS_CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  auto it = limit.find({dev, kernel});
  if (it == limit.end()) {
    cudaFuncAttributes fa;
    WEKWS_CUDA_OK(cudaFuncGetAttributes(&fa, kernel));
    it = limit.emplace(std::make_pair(dev, kernel), (size_t)fa.maxDynamicSharedSizeBytes).first;
  }
  if (it->second < bytes) {
    WEKWS_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    it->second = bytes;
  }
  return WEKWS_OK;
}

namespace {

__global__ void softmax_rows_kernel(float* x, long long rows, int n) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float* p = x + row * n;
  float m, s;
  warp_row_max_sum(p, n, lane, m, s);
  for (int i = lane; i < n; i += 32) p[i] = expf(p[i] - m) / s;
}

struct Folded {           // BN as per-channel scale/shift
  std::vector<double> s, t;
};

enum class TcKernel { None, Mdtc, Tcn, DsTcn, Gru };   // the tensor-core kernel a model has, if any

// Where one state_dict tensor sits in h_vec: `name` viewed as [rows][cols] lands transposed at h_vec[dst + c * ld + r],
// the meaning of FsmnParamCopy (fsmn.h) without its source pointer.
struct PackedParam {
  std::string name;
  long long dst;
  int rows, cols, ld;
};

}  // namespace
}  // namespace wekws

using namespace wekws;

struct wekws_model {
  wekws_model_config cfg;
  std::map<std::string, std::vector<float>> tensors;
  bool finalized = false;
  int device = 0;
  int padding = 0, padmax = 0, nblocks = 0;
  bool has_cmvn = false;
  std::vector<int> dil, coff;
  std::vector<float> h_stream, h_vec;
  std::vector<int> h_chunk_off;
  float* d_stream = nullptr;
  float* d_vec = nullptr;
  int* d_chunk_off = nullptr;
  ConvArgs conv{};
  GruArgs gru{};
  int conv_max_T = 0;
  // tensor-core path: the kernel the pack produced (None: the FP32 kernels only) and its pre-swizzled weight images
  TcKernel tc = TcKernel::None;
  std::vector<std::vector<float>> folded;   // folded GEMM weights W^T [K][C] in consumption order
  std::vector<uint8_t> h_wimg;
  uint8_t* d_wimg = nullptr;
  int precision = 0;                        // 0 auto (tensor cores where eligible), 1 fp32 FFMA only, 2 tensor cores
  TcArgs tcargs{};                          // MDTC, hidden 64
  TcnTcArgs tcnargs{};                      // dense TCN, hidden 64
  DsTcArgs dsargs{};                        // depthwise-separable TCN, hidden 256
  FsmnArgs fsmn{};                          // FSMN backbone (fsmn.cu): weights live in h_vec / d_vec
  bool cls_tc = false;                      // wide classifier head (odim > 4) as its own tensor-core GEMM (linear_tc.cu)
  std::vector<uint8_t> h_cimg;              //   behind the tensor-core DS-TCN backbone
  std::vector<float> h_cbias;
  uint8_t* d_cimg = nullptr;
  float* d_cbias = nullptr;
  float* d_hidden = nullptr;                // (B, T, 256) scratch between the two kernels; grows monotonically
  size_t hidden_cap = 0;
  GruTcArgs grutc{};                        // tensor-core GRU (gru_tc.cu): weight stream lives in h_wimg / d_wimg
  int head = WEKWS_HEAD_LINEAR;             // wekws_head; GLOBAL / LAST: the backbone kernel pools, cls_head.cu classifies
  int v_w0 = 0, v_b0 = 0, v_w1 = 0, v_b1 = 0;   // the head's MLP in h_vec (pack_head)
  float* d_pool = nullptr;                  // (B, hdim) pooled backbone output between the two kernels; grows monotonically
  size_t pool_cap = 0;
  // FSMN and GRU: every trainable parameter's place in h_vec, in wekws_train_num_params order (FSMN: state_dict,
  // GRU: named_parameters), which wekws_model_load_params packs on the device; empty for the other backbones
  std::vector<PackedParam> params;
};

namespace {

int get_tensor(const wekws_model* m, const std::string& name, size_t numel, const float** out) {
  auto it = m->tensors.find(name);
  if (it == m->tensors.end()) {
    set_error("finalize: tensor '%s' was never set", name.c_str());
    return WEKWS_ERR_STATE;
  }
  if (it->second.size() != numel) {
    set_error("finalize: tensor '%s' has %zu elements, expected %zu", name.c_str(), it->second.size(), numel);
    return WEKWS_ERR_INVALID;
  }
  *out = it->second.data();
  return WEKWS_OK;
}

#define GET(ptr, name, numel)                                            \
  const float* ptr = nullptr;                                            \
  do { int _rc = get_tensor(m, (name), (numel), &ptr); if (_rc) return _rc; } while (0)

int fold_bn(const wekws_model* m, const std::string& p, int C, Folded* f) {
  GET(g, p + ".weight", (size_t)C);
  GET(b, p + ".bias", (size_t)C);
  GET(mu, p + ".running_mean", (size_t)C);
  GET(var, p + ".running_var", (size_t)C);
  f->s.resize(C); f->t.resize(C);
  for (int c = 0; c < C; ++c) {
    const double s = (double)g[c] / sqrt((double)var[c] + 1e-5);
    f->s[c] = s;
    f->t[c] = (double)b[c] - (double)mu[c] * s;
  }
  return WEKWS_OK;
}

size_t pad4(size_t n) { return (n + 3) & ~(size_t)3; }

// Appends a zero-filled block of n floats to h_vec; returns where it starts.
int new_block(wekws_model* m, size_t n) {
  const size_t off = m->h_vec.size();
  m->h_vec.resize(off + n, 0.f);
  return (int)off;
}

// Copies the state_dict tensor `name`, viewed as [rows][cols], to h_vec[dst + c * ld + r] inside a block the caller
// has made, and appends its entry to `table` (nullptr: the model does not train on its pack).  This is what
// fsmn_pack_kernel does with the same entry on the device.
int place(wekws_model* m, std::vector<PackedParam>* table, const std::string& name, int rows, int cols, long long dst,
          int ld) {
  GET(src, name, (size_t)rows * cols);
  for (int r = 0; r < rows; ++r)
    for (int c = 0; c < cols; ++c) m->h_vec[dst + (long long)c * ld + r] = src[(size_t)r * cols + c];
  if (table) table->push_back({name, dst, rows, cols, ld});
  return WEKWS_OK;
}

#define PLACE(table, name, rows, cols, dst, ld)                                              \
  do { int _rc = place(m, (table), (name), (rows), (cols), (dst), (ld)); if (_rc) return _rc; } while (0)

// Appends W^T (K x C, from W[o][c] * s[o] with arbitrary source strides) as row chunks.
void push_gemm(wekws_model* m, int K, int C, const float* W, size_t o_stride, size_t c_stride, const double* s) {
  const int KC = conv_chunk_rows(C);
  m->folded.emplace_back((size_t)K * C);
  for (int k = 0; k < K; ++k)
    for (int o = 0; o < C; ++o)
      m->folded.back()[(size_t)k * C + o] = (float)((double)W[o * o_stride + k * c_stride] * (s ? s[o] : 1.0));
  for (int k0 = 0; k0 < K; k0 += KC) {
    const int kk = K - k0 < KC ? K - k0 : KC;
    m->h_chunk_off.push_back((int)m->h_stream.size());
    for (int k = k0; k < k0 + kk; ++k)
      for (int o = 0; o < C; ++o)
        m->h_stream.push_back((float)((double)W[o * o_stride + k * c_stride] * (s ? s[o] : 1.0)));
  }
}

int pack_common_front(wekws_model* m, int* v_mean, int* v_istd) {
  const int idim = m->cfg.idim;
  m->has_cmvn = m->tensors.count("global_cmvn.mean") != 0;
  *v_mean = (int)m->h_vec.size();
  m->h_vec.resize(m->h_vec.size() + pad4(idim), 0.f);
  *v_istd = (int)m->h_vec.size();
  m->h_vec.resize(m->h_vec.size() + pad4(idim), 1.f);
  if (m->has_cmvn) {
    GET(mean, "global_cmvn.mean", (size_t)idim);
    GET(istd, "global_cmvn.istd", (size_t)idim);
    for (int k = 0; k < idim; ++k) {
      m->h_vec[*v_mean + k] = mean[k];
      m->h_vec[*v_istd + k] = m->cfg.norm_var ? istd[k] : 1.f;   // cmvn.py:46-47
    }
  }
  return WEKWS_OK;
}

// the per-frame classifier: W_c^T [H][odim], b_c
int pack_classifier(wekws_model* m, std::vector<PackedParam>* table, int H, int* v_wc, int* v_bc) {
  const int odim = m->cfg.odim;
  *v_wc = new_block(m, pad4((size_t)H * odim));
  *v_bc = new_block(m, pad4(odim));
  PLACE(table, "classifier.linear.weight", odim, H, *v_wc, odim);
  PLACE(table, "classifier.linear.bias", odim, 1, *v_bc, 1);
  return WEKWS_OK;
}

// Utterance-level head (classifier.py:19-40 around kws_model.py:180-182): W0^T [H][64], b0, W1^T [64][odim], b1
int pack_head(wekws_model* m, int H) {
  const int odim = m->cfg.odim, W = kHeadWidth;
  m->v_w0 = new_block(m, pad4((size_t)H * W));
  m->v_b0 = new_block(m, W);
  m->v_w1 = new_block(m, pad4((size_t)W * odim));
  m->v_b1 = new_block(m, pad4(odim));
  PLACE(nullptr, "classifier.classifier.0.weight", W, H, m->v_w0, W);
  PLACE(nullptr, "classifier.classifier.0.bias", W, 1, m->v_b0, 1);
  PLACE(nullptr, "classifier.classifier.3.weight", odim, W, m->v_w1, odim);
  PLACE(nullptr, "classifier.classifier.3.bias", odim, 1, m->v_b1, 1);
  return WEKWS_OK;
}

// 16 KB slot: the K-major SWIZZLE_128B bf16 hi|lo image (tc_common.cuh) of W[n][k0 .. k0+64), n < 64, from W^T [K][64]
void write_w_image(uint8_t* dst, const std::vector<float>& wt, int K, int k0) {
  tc::write_sw128_bf16x3(dst, 64, wt.data() + (size_t)k0 * 64, 1, 64, 64, K - k0);
}

// 32 KB slot: the same for the 128 output channels n0 .. n0+127 of W^T [K][ldn] (dstcn_tc.cu)
void write_w_image128(uint8_t* dst, const std::vector<float>& wt, int ldn, int K, int k0, int n0) {
  tc::write_sw128_bf16x3(dst, 128, wt.data() + (size_t)k0 * ldn + n0, 1, ldn, 128, K - k0);
}

// 16 KB slots of the hidden-64 kernels (mdtc_tc.h, tcn_tc.h): [Wp atom0][Wp atom1], then one per folded 64 x 64 GEMM
void pack_images64(wekws_model* m) {
  const int idim = m->conv.idim, ngemm = (int)m->folded.size() - 1;
  m->h_wimg.assign((size_t)(2 + ngemm) * 16384, 0);
  write_w_image(m->h_wimg.data(), m->folded[0], idim, 0);
  if (idim > 64) write_w_image(m->h_wimg.data() + 16384, m->folded[0], idim, 64);
  for (int g = 0; g < ngemm; ++g) write_w_image(m->h_wimg.data() + (size_t)(2 + g) * 16384, m->folded[1 + g], 64, 0);
}

// the ConvArgs fields every tensor-core conv argument block repeats (TcArgs, TcnTcArgs, DsTcArgs)
template <class A>
void init_tc_args(A* t, const ConvArgs& a) {
  memset(t, 0, sizeof(*t));
  t->idim = a.idim; t->odim = a.odim; t->nblocks = a.nblocks; t->ktaps = a.ktaps; t->P = a.P;
  t->act = a.act; t->has_cmvn = a.has_cmvn;
  t->v_mean = a.v_mean; t->v_istd = a.v_istd; t->v_bp = a.v_bp; t->v_blocks = a.v_blocks;
  t->v_blk_stride = a.v_blk_stride; t->v_wc = a.v_wc; t->v_bc = a.v_bc;
  for (int b = 0; b < a.nblocks; ++b) { t->dil[b] = a.dil[b]; t->coff[b] = a.coff[b]; }
}

// Tensor-core eligibility + pre-swizzled bf16x3 weight images (mdtc_tc.cu, tcn_tc.cu, dstcn_tc.cu); sets m->tc
void pack_tc(wekws_model* m) {
  m->tc = TcKernel::None;
  m->cls_tc = false;
  m->h_wimg.clear();
  m->h_cimg.clear();
  const wekws_model_config& c = m->cfg;
  const ConvArgs& a = m->conv;
  const bool head = m->head != WEKWS_HEAD_LINEAR;
  if (head && c.backbone != WEKWS_BACKBONE_MDTC) return;     // TCN / DS-TCN heads run on the FP32 conv kernel
  if (c.backbone == WEKWS_BACKBONE_DSTCN) {
    init_tc_args(&m->dsargs, a);
    // output_dim > 4 (CTC vocabularies): the classifier becomes its own tensor-core GEMM fed from a hidden scratch
    const bool cls_tc = c.odim > 4 && linear_tc_eligible(c.odim, c.hdim);
    if (!dstcn_tc_eligible(m->dsargs, c.hdim, cls_tc) || m->folded.size() != (size_t)(1 + a.nblocks)) return;
    m->cls_tc = cls_tc;
    if (cls_tc) {           // W_c^T [256][odim] sits in h_vec at v_wc (pack_classifier), the bias at v_bc
      m->h_cimg.assign(linear_tc_image_bytes(c.odim, c.hdim), 0);
      linear_tc_pack(m->h_cimg.data(), m->h_vec.data() + a.v_wc, c.odim, c.odim, c.hdim);
      m->h_cbias.assign((size_t)((c.odim + 127) / 128) * 128, 0.f);
      for (int j = 0; j < c.odim; ++j) m->h_cbias[j] = m->h_vec[a.v_bc + j];
    }
    const int natoms = (a.idim + 63) / 64;
    m->h_wimg.assign((size_t)(2 * natoms + 8 * a.nblocks) * 32768, 0);
    uint8_t* dst = m->h_wimg.data();
    for (int at = 0; at < natoms; ++at)
      for (int h = 0; h < 2; ++h, dst += 32768) write_w_image128(dst, m->folded[0], 256, a.idim, 64 * at, 128 * h);
    for (int b = 0; b < a.nblocks; ++b)
      for (int ks = 0; ks < 4; ++ks)
        for (int h = 0; h < 2; ++h, dst += 32768) write_w_image128(dst, m->folded[1 + b], 256, 256, 64 * ks, 128 * h);
    m->tc = TcKernel::DsTcn;
    return;
  }
  if (c.backbone == WEKWS_BACKBONE_TCN && c.hdim == 64) {
    init_tc_args(&m->tcnargs, a);
    if (!tcn_tc_eligible(m->tcnargs, m->padmax) || m->folded.size() != (size_t)(1 + a.ktaps * a.nblocks)) return;
    pack_images64(m);
    m->tc = TcKernel::Tcn;
    return;
  }
  if (c.backbone != WEKWS_BACKBONE_MDTC || c.hdim != 64) return;
  TcArgs& t = m->tcargs;
  init_tc_args(&t, a);
  t.stack_size = a.stack_size;
  if (!tc_eligible(t, m->padmax, head) || m->folded.size() != (size_t)(1 + 2 * a.nblocks)) return;
  pack_images64(m);
  // depthwise taps + the two GEMM biases of every block, passed by value with the launch (mdtc_tc.h TcArgs::cw)
  for (int b = 0; b < a.nblocks; ++b) {
    const float* vb = m->h_vec.data() + a.v_blocks + (size_t)b * a.v_blk_stride;
    float* dst = reinterpret_cast<float*>(&t.cw[b][0]);
    for (int j = 0; j < 5; ++j)
      for (int ch = 0; ch < 64; ++ch) dst[j * 64 + ch] = j < a.ktaps ? vb[j * 64 + ch] : 0.f;
    // the folded depthwise bias goes through the pointwise-1 matrix into b1 (h = relu(W1 (dw + b_dw) + b1)), so the
    // depthwise loop of the kernel starts from zero instead of loading a per-channel bias
    const float* w1t = m->folded[1 + 2 * b].data();     // W1^T [k][n]
    const float* bdw = vb + a.ktaps * 64;
    for (int ch = 0; ch < 64; ++ch) {
      double acc = vb[(a.ktaps + 1) * 64 + ch];
      for (int k = 0; k < 64; ++k) acc += (double)w1t[(size_t)k * 64 + ch] * (double)bdw[k];
      dst[5 * 64 + ch] = (float)acc;
      dst[6 * 64 + ch] = vb[(a.ktaps + 2) * 64 + ch];
    }
  }
  m->tc = TcKernel::Mdtc;
}

int pack_conv(wekws_model* m) {
  const wekws_model_config& c = m->cfg;
  const int C = c.hdim, K = c.kernel_size, idim = c.idim;
  WEKWS_REQUIRE(C == 32 || C == 64 || C == 128 || C == 256, "hidden_dim %d unsupported (32/64/128/256)", C);
  WEKWS_REQUIRE(K >= 2 && K <= 8, "kernel_size %d unsupported (2..8)", K);
  WEKWS_REQUIRE(idim >= 1 && idim <= 128, "input_dim %d unsupported (1..128)", idim);
  std::vector<std::string> prefix;
  m->dil.clear(); m->coff.clear();
  if (c.backbone == WEKWS_BACKBONE_MDTC) {
    WEKWS_REQUIRE(c.num_stack >= 1 && c.stack_size >= 1, "mdtc: num_stack/stack_size must be >= 1");
    prefix.push_back("backbone.preprocessor");
    m->dil.push_back(1);
    for (int s = 0; s < c.num_stack; ++s)
      for (int l = 0; l < c.stack_size; ++l) {
        prefix.push_back("backbone.blocks." + std::to_string(s) + ".res_blocks." + std::to_string(l));
        m->dil.push_back(1 << l);
      }
  } else {
    WEKWS_REQUIRE(c.num_layers >= 1, "tcn: num_layers must be >= 1");
    for (int i = 0; i < c.num_layers; ++i) {
      prefix.push_back("backbone.network." + std::to_string(i) + ".cnn");
      m->dil.push_back(1 << i);
    }
  }
  m->nblocks = (int)prefix.size();
  WEKWS_REQUIRE(m->nblocks <= kMaxBlocks, "%d blocks exceed the supported %d", m->nblocks, kMaxBlocks);
  m->padding = 0; m->padmax = 0;
  for (int b = 0; b < m->nblocks; ++b) {
    m->coff.push_back(m->padding);
    const int pad = m->dil[b] * (K - 1);
    m->padding += pad;
    if (pad > m->padmax) m->padmax = pad;
  }
  m->h_stream.clear(); m->h_vec.clear(); m->h_chunk_off.clear(); m->folded.clear();
  ConvArgs& a = m->conv;
  memset(&a, 0, sizeof(a));
  int rc = pack_common_front(m, &a.v_mean, &a.v_istd);
  if (rc) return rc;
  // preprocessing Linear (subsampling.py:45-48): W (C, idim)
  {
    GET(w, "preprocessing.out.0.weight", (size_t)C * idim);
    GET(b, "preprocessing.out.0.bias", (size_t)C);
    push_gemm(m, idim, C, w, idim, 1, nullptr);
    a.v_bp = (int)m->h_vec.size();
    m->h_vec.insert(m->h_vec.end(), b, b + C);
  }
  a.v_blocks = (int)m->h_vec.size();
  a.v_blk_stride = c.backbone == WEKWS_BACKBONE_MDTC ? (K + 3) * C
                 : c.backbone == WEKWS_BACKBONE_DSTCN ? (K + 2) * C : C;
  for (int bi = 0; bi < m->nblocks; ++bi) {
    const std::string& p = prefix[bi];
    const size_t v0 = m->h_vec.size();
    if (c.backbone == WEKWS_BACKBONE_MDTC || c.backbone == WEKWS_BACKBONE_DSTCN) {
      const bool md = c.backbone == WEKWS_BACKBONE_MDTC;
      const std::string dw = md ? p + ".conv1.conv" : p + ".0";
      const std::string dwbn = md ? p + ".conv1.bn" : p + ".1";
      const std::string pw = md ? p + ".conv1.pointwise" : p + ".3";
      const std::string pwbn = md ? p + ".bn1" : p + ".4";
      GET(wd, dw + ".weight", (size_t)C * K);
      GET(bd, dw + ".bias", (size_t)C);
      Folded f0, f1;
      if ((rc = fold_bn(m, dwbn, C, &f0))) return rc;
      if ((rc = fold_bn(m, pwbn, C, &f1))) return rc;
      for (int j = 0; j < K; ++j)
        for (int ch = 0; ch < C; ++ch) m->h_vec.push_back((float)((double)wd[ch * K + j] * f0.s[ch]));
      for (int ch = 0; ch < C; ++ch) m->h_vec.push_back((float)((double)bd[ch] * f0.s[ch] + f0.t[ch]));
      GET(w1, pw + ".weight", (size_t)C * C);
      GET(b1, pw + ".bias", (size_t)C);
      push_gemm(m, C, C, w1, C, 1, f1.s.data());
      for (int o = 0; o < C; ++o) m->h_vec.push_back((float)((double)b1[o] * f1.s[o] + f1.t[o]));
      if (md) {
        Folded f2;
        if ((rc = fold_bn(m, p + ".bn2", C, &f2))) return rc;
        GET(w2, p + ".conv2.weight", (size_t)C * C);
        GET(b2, p + ".conv2.bias", (size_t)C);
        push_gemm(m, C, C, w2, C, 1, f2.s.data());
        for (int o = 0; o < C; ++o) m->h_vec.push_back((float)((double)b2[o] * f2.s[o] + f2.t[o]));
      }
    } else {  // dense TCN: weight (C, C, K) -> K tap matrices
      GET(w, p + ".0.weight", (size_t)C * C * K);
      GET(b, p + ".0.bias", (size_t)C);
      Folded f;
      if ((rc = fold_bn(m, p + ".1", C, &f))) return rc;
      for (int j = 0; j < K; ++j) push_gemm(m, C, C, w + j, (size_t)C * K, K, f.s.data());
      for (int o = 0; o < C; ++o) m->h_vec.push_back((float)((double)b[o] * f.s[o] + f.t[o]));
    }
    if (m->h_vec.size() - v0 != (size_t)a.v_blk_stride) {
      set_error("internal: block vector stride mismatch");
      return WEKWS_ERR_INVALID;
    }
  }
  if (m->head != WEKWS_HEAD_LINEAR) {
    if ((rc = pack_head(m, C))) return rc;
  } else if ((rc = pack_classifier(m, nullptr, C, &a.v_wc, &a.v_bc))) {
    return rc;
  }
  m->h_chunk_off.push_back((int)m->h_stream.size());
  a.kind = c.backbone; a.C = C; a.idim = idim; a.odim = c.odim; a.nblocks = m->nblocks; a.ktaps = K;
  a.P = m->padding; a.stack_size = c.stack_size > 0 ? c.stack_size : 1; a.act = c.activation;
  a.has_cmvn = m->has_cmvn ? 1 : 0;
  a.n_chunks = (int)m->h_chunk_off.size() - 1;
  for (int b = 0; b < m->nblocks; ++b) { a.dil[b] = m->dil[b]; a.coff[b] = m->coff[b]; }
  pack_tc(m);
  return WEKWS_OK;
}

int pack_gru(wekws_model* m) {
  const wekws_model_config& c = m->cfg;
  const int H = c.hdim, G = 3 * H, idim = c.idim, L = c.num_layers;
  WEKWS_REQUIRE(H == 128, "GRU hidden_dim %d unsupported (128 only)", H);
  WEKWS_REQUIRE(L >= 1 && L <= 4, "GRU num_layers %d unsupported (1..4)", L);
  WEKWS_REQUIRE(idim >= 1 && idim <= 128, "input_dim %d unsupported (1..128)", idim);
  m->h_stream.clear(); m->h_vec.clear(); m->h_chunk_off.clear();
  m->padding = 0; m->padmax = 0; m->nblocks = L;
  GruArgs& a = m->gru;
  memset(&a, 0, sizeof(a));
  int rc = pack_common_front(m, &a.v_mean, &a.v_istd);
  if (rc) return rc;
  std::vector<PackedParam>* tab = &m->params;
  a.v_wp = new_block(m, (size_t)idim * H);
  a.v_bp = new_block(m, H);
  PLACE(tab, "preprocessing.out.0.weight", H, idim, a.v_wp, H);
  PLACE(tab, "preprocessing.out.0.bias", H, 1, a.v_bp, 1);
  a.v_layers = (int)m->h_vec.size();
  a.v_layer_stride = 2 * H * G + 2 * G;
  for (int l = 0; l < L; ++l) {
    const std::string sfx = "_l" + std::to_string(l);
    // row k: [W_ih[:, k] | W_hh[:, k]]  (768 floats, streamed by TMA), then b_ih, b_hh
    const long long base = new_block(m, a.v_layer_stride);
    PLACE(tab, "backbone.weight_ih" + sfx, G, H, base, 2 * G);
    PLACE(tab, "backbone.weight_hh" + sfx, G, H, base + G, 2 * G);
    PLACE(tab, "backbone.bias_ih" + sfx, G, 1, base + 2LL * H * G, 1);
    PLACE(tab, "backbone.bias_hh" + sfx, G, 1, base + 2LL * H * G + G, 1);
  }
  if ((rc = pack_classifier(m, tab, H, &a.v_wc, &a.v_bc))) return rc;
  a.L = L; a.H = H; a.idim = idim; a.odim = c.odim; a.act = c.activation; a.has_cmvn = m->has_cmvn ? 1 : 0;
  // tensor-core variant: the per-step weight stream as pre-swizzled bf16 hi|lo operand chunks
  m->tc = TcKernel::None;
  m->h_wimg.clear();
  if (gru_tc_eligible(L, H, idim)) {
    GET(wp, "preprocessing.out.0.weight", (size_t)H * idim);
    const float* wih[4];
    const float* whh[4];
    for (int l = 0; l < L; ++l) {
      const std::string sfx = "_l" + std::to_string(l);
      if ((rc = get_tensor(m, "backbone.weight_ih" + sfx, (size_t)G * H, &wih[l]))) return rc;
      if ((rc = get_tensor(m, "backbone.weight_hh" + sfx, (size_t)G * H, &whh[l]))) return rc;
    }
    m->h_wimg.assign(gru_tc_image_bytes(L, idim), 0);
    gru_tc_pack(m->h_wimg.data(), wp, idim, wih, whh, L);
    GruTcArgs& t = m->grutc;
    memset(&t, 0, sizeof(t));
    t.L = L; t.idim = idim; t.odim = c.odim; t.act = c.activation; t.has_cmvn = a.has_cmvn;
    t.v_mean = a.v_mean; t.v_istd = a.v_istd; t.v_bp = a.v_bp; t.v_layers = a.v_layers;
    t.v_layer_stride = a.v_layer_stride; t.v_wc = a.v_wc; t.v_bc = a.v_bc;
    m->tc = TcKernel::Gru;
  }
  return WEKWS_OK;
}


// FSMN (wekws/model/fsmn.py:401-495): every matrix transposed to [K][Npad] (Npad = N rounded up to the GEMM pass width,
// zero filled) so the kernel streams K-chunks with 16-byte cp.async; biases padded the same way; memory taps as
// [lorder + rorder][proj] (left taps, then right taps).
int pack_fsmn(wekws_model* m) {
  const wekws_model_config& c = m->cfg;
  const int idim = c.idim, A1 = c.fsmn_input_affine_dim, D = c.fsmn_linear_dim, P = c.fsmn_proj_dim;
  const int A2 = c.fsmn_output_affine_dim, O = c.odim, L = c.num_layers, lo = c.fsmn_left_order, ro = c.fsmn_right_order;
  WEKWS_REQUIRE(idim >= 1 && A1 >= 1 && D >= 1 && P >= 1 && A2 >= 1 && L >= 1 && L <= 16, "fsmn: bad layer dimensions");
  WEKWS_REQUIRE(lo >= 1 && ro >= 1, "fsmn: left_order %d / right_order %d unsupported (the reference's FSMNBlock itself "
                "breaks for right_order = 0: fsmn.py:235 slices x_pad[:, :, :-0])", lo, ro);
  m->h_stream.clear(); m->h_vec.clear(); m->h_chunk_off.clear();
  m->padding = lo - 1 + ro; m->padmax = m->padding; m->nblocks = L;
  FsmnArgs& a = m->fsmn;
  memset(&a, 0, sizeof(a));
  int rc = pack_common_front(m, &a.o_mean, &a.o_istd);
  if (rc) return rc;
  const int NP = fsmn_pass_cols();
  auto npad = [&](int n) { return (n + NP - 1) / NP * NP; };
  std::vector<PackedParam>* tab = &m->params;
  // the state_dict Linear `p` ([N][K], with its bias [N] unless o_b is null) -> W^T [K][npad(N)] at o_w, b at o_b
  auto push_linear = [&](const std::string& p, int N, int K, int* o_w, int* o_b) -> int {
    *o_w = new_block(m, (size_t)K * npad(N));
    PLACE(tab, p + ".weight", N, K, *o_w, npad(N));
    if (o_b) {
      *o_b = new_block(m, npad(N));
      PLACE(tab, p + ".bias", N, 1, *o_b, 1);
    }
    return WEKWS_OK;
  };
  if ((rc = push_linear("backbone.in_linear1.linear", A1, idim, &a.o_w_in1, &a.o_b_in1)) ||
      (rc = push_linear("backbone.in_linear2.linear", D, A1, &a.o_w_in2, &a.o_b_in2)))
    return rc;
  a.o_layers = (int)m->h_vec.size();
  for (int l = 0; l < L; ++l) {
    const std::string p = "backbone.fsmn." + std::to_string(l) + ".";
    const int base = (int)m->h_vec.size();
    int o_wp, o_wa, o_ba;
    if ((rc = push_linear(p + "0.linear", P, D, &o_wp, nullptr))) return rc;
    const int o_taps = new_block(m, pad4((size_t)(lo + ro) * P));
    PLACE(tab, p + "1.conv_left.weight", P, lo, o_taps, P);
    PLACE(tab, p + "1.conv_right.weight", P, ro, o_taps + (long long)lo * P, P);
    if ((rc = push_linear(p + "2.linear", D, P, &o_wa, &o_ba))) return rc;
    if (l == 0) {
      a.lo_wp = o_wp - base; a.lo_taps = o_taps - base; a.lo_wa = o_wa - base; a.lo_ba = o_ba - base;
      a.layer_stride = (int)m->h_vec.size() - base;
    }
  }
  if ((rc = push_linear("backbone.out_linear1.linear", A2, D, &a.o_w_out1, &a.o_b_out1)) ||
      (rc = push_linear("backbone.out_linear2.linear", O, A2, &a.o_w_out2, &a.o_b_out2)))
    return rc;
  a.idim = idim; a.aff_in = A1; a.lin = D; a.proj = P; a.aff_out = A2; a.odim = O; a.L = L; a.lorder = lo; a.rorder = ro;
  a.act = c.activation; a.has_cmvn = m->has_cmvn ? 1 : 0; a.norm_var = 1;      // istd already 1 when norm_var is off
  a.np_aff_in = npad(A1); a.np_lin = npad(D); a.np_proj = npad(P); a.np_aff_out = npad(A2); a.np_odim = npad(O);
  const int m0 = idim > D ? idim : D;
  int m1 = A1 > P ? A1 : P;
  if (A2 > m1) m1 = A2;
  a.sp0 = (int)pad4(m0) + 4; a.sp1 = (int)pad4(m1) + 4; a.spm = (int)pad4(P) + 4;   // +4: rows start in different banks
  WEKWS_REQUIRE(fsmn_smem_bytes(a) <= 226 * 1024, "fsmn: layer widths (%d, %d, %d) exceed the fused kernel's shared memory", m0, m1, P);
  return WEKWS_OK;
}

void free_device(wekws_model* m) {
  cudaFree(m->d_stream); cudaFree(m->d_vec); cudaFree(m->d_chunk_off); cudaFree(m->d_wimg);
  cudaFree(m->d_cimg); cudaFree(m->d_cbias); cudaFree(m->d_hidden); cudaFree(m->d_pool);
  m->d_stream = nullptr; m->d_vec = nullptr; m->d_chunk_off = nullptr; m->d_wimg = nullptr;
  m->d_cimg = nullptr; m->d_cbias = nullptr; m->d_hidden = nullptr; m->hidden_cap = 0;
  m->d_pool = nullptr; m->pool_cap = 0;
}

template <class T>
int upload(T** d_dst, const std::vector<T>& h_src) {
  WEKWS_CUDA_OK(cudaMalloc((void**)d_dst, h_src.size() * sizeof(T)));
  WEKWS_CUDA_OK(cudaMemcpy(*d_dst, h_src.data(), h_src.size() * sizeof(T), cudaMemcpyHostToDevice));
  return WEKWS_OK;
}

// grows a scratch buffer to at least `need` floats; contents are not kept
int grow_scratch(float** buf, size_t* cap, size_t need, cudaStream_t st) {
  if (need <= *cap) return WEKWS_OK;
  WEKWS_CUDA_OK(cudaStreamSynchronize(st));          // the old scratch may still be in use on this stream
  cudaFree(*buf);
  *buf = nullptr; *cap = 0;
  WEKWS_CUDA_OK(cudaMalloc((void**)buf, need * sizeof(float)));
  *cap = need;
  return WEKWS_OK;
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// The kernel a forward call of B streams x T frames takes: the model's tensor-core kernel unless the precision mode,
// the shape or the pointers rule it out, else TcKernel::None (the FP32 kernel).  feats_aligned: the features are
// 16-byte aligned; caches_aligned: so are out_cache and in_cache (if given).
TcKernel select_kernel(const wekws_model* m, int64_t B, int64_t T, bool feats_aligned, bool caches_aligned) {
  if (m->tc == TcKernel::None || m->precision == 1) return TcKernel::None;
  if (m->tc == TcKernel::Gru) {
    // which GRU kernel is faster depends on the batch as well: the weight-streaming tensor-core kernel takes about the
    // same time per step whatever the batch (up to one 64-stream tile per SM), the FP32 kernel scales with the streams
    // per SM and has the shorter single-step latency at small batches
    const bool tc = T >= 1 && (m->precision == 2 || B >= (T == 1 ? 640 : T < 8 ? 400 : 256));
    return tc ? TcKernel::Gru : TcKernel::None;
  }
  // conv backbones: chunks of >= 8 frames; MDTC also reads and writes the cache rows with 16-byte accesses
  const bool aligned = feats_aligned && (m->tc != TcKernel::Mdtc || caches_aligned);
  return T >= 8 && aligned ? m->tc : TcKernel::None;
}

}  // namespace

// ------------------------------------------------------------------------------- C ABI
extern "C" const char* wekws_last_error(void) { return tl_error.c_str(); }
extern "C" int wekws_abi_version(void) { return WEKWS_B200_ABI_VERSION; }
extern "C" uint64_t wekws_launch_count(void) { return g_launches.load(); }

extern "C" int wekws_model_create(const wekws_model_config* cfg, wekws_model** out) {
  WEKWS_REQUIRE(cfg && out, "wekws_model_create: null argument");
  WEKWS_REQUIRE(cfg->backbone >= WEKWS_BACKBONE_MDTC && cfg->backbone <= WEKWS_BACKBONE_FSMN,
                "unknown backbone id %d", cfg->backbone);
  WEKWS_REQUIRE(cfg->odim >= 1, "output_dim must be >= 1");
  WEKWS_REQUIRE(cfg->activation == WEKWS_ACT_IDENTITY || cfg->activation == WEKWS_ACT_SIGMOID,
                "unknown activation id %d", cfg->activation);
  wekws_model* m = new (std::nothrow) wekws_model();
  if (!m) { set_error("out of host memory"); return WEKWS_ERR_NOMEM; }
  m->cfg = *cfg;
  *out = m;
  return WEKWS_OK;
}

extern "C" void wekws_model_destroy(wekws_model* m) {
  if (!m) return;
  free_device(m);
  delete m;
}

extern "C" int wekws_model_padding(const wekws_model* m) {
  if (!m) return 0;
  if (m->cfg.backbone == WEKWS_BACKBONE_GRU) return 0;
  if (m->cfg.backbone == WEKWS_BACKBONE_FSMN) return m->cfg.fsmn_left_order - 1 + m->cfg.fsmn_right_order;
  int pad = 0;
  const int K = m->cfg.kernel_size;
  if (m->cfg.backbone == WEKWS_BACKBONE_MDTC) {
    pad = K - 1;
    for (int s = 0; s < m->cfg.num_stack; ++s)
      for (int l = 0; l < m->cfg.stack_size; ++l) pad += (1 << l) * (K - 1);
  } else {
    for (int i = 0; i < m->cfg.num_layers; ++i) pad += (1 << i) * (K - 1);
  }
  return pad;
}

extern "C" int wekws_model_set_tensor(wekws_model* m, const char* name, const float* h_data, int64_t numel) {
  WEKWS_REQUIRE(m && name && (h_data || numel == 0) && numel >= 0, "wekws_model_set_tensor: bad argument");
  m->tensors[name].assign(h_data, h_data + numel);
  m->finalized = false;
  return WEKWS_OK;
}

extern "C" int wekws_model_set_head(wekws_model* m, int head) {
  WEKWS_REQUIRE(m, "wekws_model_set_head: null handle");
  WEKWS_REQUIRE(head >= WEKWS_HEAD_LINEAR && head <= WEKWS_HEAD_LAST, "unknown head id %d", head);
  WEKWS_REQUIRE(head == WEKWS_HEAD_LINEAR || m->cfg.backbone == WEKWS_BACKBONE_MDTC ||
                m->cfg.backbone == WEKWS_BACKBONE_TCN || m->cfg.backbone == WEKWS_BACKBONE_DSTCN,
                "the %s head is implemented behind the MDTC, TCN and DS-TCN backbones only",
                head == WEKWS_HEAD_GLOBAL ? "global" : "last");
  m->head = head;
  m->finalized = false;
  return WEKWS_OK;
}

extern "C" int wekws_model_pack(wekws_model* m) {
  WEKWS_REQUIRE(m, "wekws_model_pack: null handle");
  m->params.clear();
  if (m->cfg.backbone == WEKWS_BACKBONE_FSMN) return pack_fsmn(m);
  return m->cfg.backbone == WEKWS_BACKBONE_GRU ? pack_gru(m) : pack_conv(m);
}

extern "C" int wekws_model_finalize(wekws_model* m) {
  WEKWS_REQUIRE(m, "wekws_model_finalize: null handle");
  m->finalized = false;
  int rc = wekws_model_pack(m);
  if (rc) return rc;
  const bool conv = m->cfg.backbone != WEKWS_BACKBONE_FSMN && m->cfg.backbone != WEKWS_BACKBONE_GRU;
  if (conv) {
    // every conv model keeps the FP32 kernel (T < 8, precision "fp32", misaligned inputs), so its one-frame tile with
    // the widest cache slice must fit in shared memory, whatever tensor-core kernel the model also has
    m->conv_max_T = conv_backbone_max_T(m->conv, m->padmax);
    WEKWS_REQUIRE(m->conv_max_T >= 1, "model does not fit the FP32 conv kernel's shared memory: hidden %d with a "
                  "widest cache slice of %d frames (dilation x (kernel_size - 1)) leaves no room for one frame",
                  m->cfg.hdim, m->padmax);
  }
  free_device(m);
  WEKWS_CUDA_OK(cudaGetDevice(&m->device));
  if ((rc = upload(&m->d_vec, m->h_vec))) return rc;
  if (m->tc != TcKernel::None && (rc = upload(&m->d_wimg, m->h_wimg))) return rc;
  if (m->cfg.backbone == WEKWS_BACKBONE_FSMN) {
    m->fsmn.w = m->d_vec;
  } else if (conv) {
    if ((rc = upload(&m->d_stream, m->h_stream))) return rc;
    if ((rc = upload(&m->d_chunk_off, m->h_chunk_off))) return rc;
    m->conv.wstream = m->d_stream; m->conv.chunk_off = m->d_chunk_off; m->conv.vec = m->d_vec;
    m->tcargs.wimg = m->d_wimg; m->tcargs.vec = m->d_vec;
    m->tcnargs.wimg = m->d_wimg; m->tcnargs.vec = m->d_vec;
    m->dsargs.wimg = m->d_wimg; m->dsargs.vec = m->d_vec;
    if (m->cls_tc) {
      if ((rc = upload(&m->d_cimg, m->h_cimg))) return rc;
      if ((rc = upload(&m->d_cbias, m->h_cbias))) return rc;
    }
  } else {
    m->gru.vec = m->d_vec;
    m->grutc.vec = m->d_vec; m->grutc.wimg = m->d_wimg;
  }
  m->finalized = true;
  return WEKWS_OK;
}

extern "C" int wekws_model_set_precision(wekws_model* m, int mode) {
  WEKWS_REQUIRE(m && mode >= 0 && mode <= 2, "wekws_model_set_precision: mode must be 0 (auto), 1 (fp32) or 2 (tensor cores wherever a kernel exists)");
  m->precision = mode;
  return WEKWS_OK;
}

extern "C" int wekws_model_uses_tensor_cores_bt(const wekws_model* m, int64_t B, int64_t T) {
  if (!m || !m->finalized) return 0;
  return select_kernel(m, B, T, true, true) != TcKernel::None ? 1 : 0;
}

extern "C" int wekws_model_uses_tensor_cores(const wekws_model* m, int64_t T) {
  return wekws_model_uses_tensor_cores_bt(m, 1 << 20, T);     // "for a large batch"
}

extern "C" int64_t wekws_model_packed_floats(const wekws_model* m, int which) {
  if (!m) return 0;
  if (which == 2) return (int64_t)(m->h_wimg.size() / sizeof(float));     // tensor-core weight images, raw bytes
  return which == 0 ? (int64_t)m->h_stream.size() : (int64_t)m->h_vec.size();
}

extern "C" int wekws_model_packed_copy(const wekws_model* m, int which, float* h_dst, int64_t capacity) {
  WEKWS_REQUIRE(m && h_dst, "wekws_model_packed_copy: null argument");
  if (which == 2) {
    WEKWS_REQUIRE((int64_t)(m->h_wimg.size() / sizeof(float)) <= capacity, "wekws_model_packed_copy: capacity too small");
    memcpy(h_dst, m->h_wimg.data(), m->h_wimg.size());
    return WEKWS_OK;
  }
  const std::vector<float>& v = which == 0 ? m->h_stream : m->h_vec;
  WEKWS_REQUIRE((int64_t)v.size() <= capacity, "wekws_model_packed_copy: capacity too small");
  memcpy(h_dst, v.data(), v.size() * sizeof(float));
  return WEKWS_OK;
}

extern "C" int wekws_model_forward(wekws_model* m, const float* d_feats, const float* d_in_cache,
                                   float* d_out, float* d_out_cache, int64_t B, int64_t T,
                                   uint32_t flags, void* stream) {
  WEKWS_REQUIRE(m, "wekws_model_forward: null handle");
  if (!m->finalized) { set_error("wekws_model_forward called before wekws_model_finalize"); return WEKWS_ERR_STATE; }
  WEKWS_REQUIRE(B >= 0 && T >= 0 && B < (1 << 30) && T < (1 << 30), "wekws_model_forward: bad B/T");
  if (B == 0 || T == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_feats && d_out && d_out_cache, "wekws_model_forward: null tensor");
  int dev = 0;
  WEKWS_CUDA_OK(cudaGetDevice(&dev));
  WEKWS_REQUIRE(dev == m->device, "model was finalized on device %d but current device is %d", m->device, dev);
  cudaStream_t st = (cudaStream_t)stream;
  const bool head = m->head != WEKWS_HEAD_LINEAR;
  const TcKernel k = select_kernel(m, B, T, aligned16(d_feats),
                                   aligned16(d_out_cache) && (d_in_cache == nullptr || aligned16(d_in_cache)));
  int rc = WEKWS_OK;
  if (m->cfg.backbone == WEKWS_BACKBONE_GRU) {
    if (k == TcKernel::Gru) {
      GruTcArgs a = m->grutc;
      a.feats = d_feats; a.in_cache = d_in_cache; a.out = d_out; a.out_cache = d_out_cache;
      a.B = (int)B; a.T = (int)T;
      rc = gru_tc_launch(a, st);
    } else {
      GruArgs a = m->gru;
      a.feats = d_feats; a.in_cache = d_in_cache; a.out = d_out; a.out_cache = d_out_cache;
      a.B = (int)B; a.T = (int)T;
      rc = gru_launch(a, st);
    }
    if (rc) return rc;
  } else {
    // time-chunk long inputs to the kernel's tile height; the cache carries the state between chunks exactly as in
    // streaming use (chunked == full utterance, SURVEY.md 8a "Numerical facts")
    const bool fsmn = m->cfg.backbone == WEKWS_BACKBONE_FSMN;
    const int maxT = fsmn ? fsmn_tile_rows() : k == TcKernel::Mdtc ? tc_max_T() : k == TcKernel::Tcn ? tcn_tc_max_T(m->padmax)
                   : k == TcKernel::DsTcn ? dstcn_tc_max_T() : m->conv_max_T;
    const bool cls_gemm = k == TcKernel::DsTcn && m->cls_tc;      // the classifier runs after the backbone, on d_hidden
    // scratch between the backbone kernel and the one that follows: pooled vectors (head), hidden rows (cls_gemm)
    if (head && (rc = grow_scratch(&m->d_pool, &m->pool_cap, (size_t)B * m->cfg.hdim, st))) return rc;
    if (cls_gemm && (rc = grow_scratch(&m->d_hidden, &m->hidden_cap, (size_t)B * T * m->cfg.hdim, st))) return rc;
    const int nchunk = (int)((T + maxT - 1) / maxT);
    const int Tc = (int)((T + nchunk - 1) / nchunk);
    for (int64_t t0 = 0; t0 < T; t0 += Tc) {
      const int Tk = (int)(T - t0 < Tc ? T - t0 : Tc);
      // head: the frames of this chunk the pooled vector takes (every frame, or the call's last one) and whether the
      // chunk stores the vector (the first chunk that contributes) or adds to it
      int pool_t0 = 0, pool_t1 = 0, pool_add = 0;
      if (m->head == WEKWS_HEAD_GLOBAL) { pool_t1 = Tk; pool_add = t0 > 0; }
      else if (m->head == WEKWS_HEAD_LAST && t0 + Tk == T) { pool_t0 = Tk - 1; pool_t1 = Tk; }
      // the model's argument block with this chunk's call fields
      auto chunk = [&](auto a) {
        using A = decltype(a);
        a.feats = d_feats + t0 * m->cfg.idim;
        a.out = d_out + t0 * m->cfg.odim;
        a.in_cache = t0 == 0 ? d_in_cache : d_out_cache;
        a.out_cache = d_out_cache;
        a.B = (int)B;
        a.T = Tk;
        a.feat_bstride = T * m->cfg.idim;
        a.out_bstride = T * m->cfg.odim;
        if constexpr (std::is_same_v<A, TcArgs> || std::is_same_v<A, ConvArgs>) {
          a.pool = head ? m->d_pool : nullptr; a.pool_t0 = pool_t0; a.pool_t1 = pool_t1; a.pool_add = pool_add;
        }
        if constexpr (std::is_same_v<A, DsTcArgs>) {
          if (cls_gemm) { a.hidden = m->d_hidden + t0 * m->cfg.hdim; a.hidden_bstride = T * m->cfg.hdim; }
        }
        return a;
      };
      switch (k) {
        case TcKernel::Mdtc: rc = mdtc_tc_launch(chunk(m->tcargs), m->padmax, st, head); break;
        case TcKernel::Tcn: rc = tcn_tc_launch(chunk(m->tcnargs), m->padmax, st); break;
        case TcKernel::DsTcn: rc = dstcn_tc_launch(chunk(m->dsargs), st); break;
        default: rc = fsmn ? fsmn_launch(chunk(m->fsmn), st) : conv_backbone_launch(chunk(m->conv), m->padmax, st);
      }
      if (rc) return rc;
    }
    if (cls_gemm) {
      // classifier (+ activation) of all B*T frames in one tensor-core GEMM over the hidden scratch (classifier.py:63-67)
      LinearTcArgs a;
      a.x = m->d_hidden; a.out = d_out; a.wimg = m->d_cimg; a.bias = m->d_cbias;
      a.rows = B * T; a.x_stride = m->cfg.hdim; a.out_stride = m->cfg.odim;
      a.N = m->cfg.odim; a.K = m->cfg.hdim; a.act = m->cfg.activation; a.n_mtiles = 0;
      if ((rc = linear_tc_launch(a, st))) return rc;
    }
  }
  if (head) {
    // MLP head (+ activation, + softmax) on the pooled vectors: (B, odim)
    ClsHeadArgs a;
    a.pool = m->d_pool; a.out = d_out; a.vec = m->d_vec;
    a.B = (int)B; a.H = m->cfg.hdim; a.odim = m->cfg.odim; a.act = m->cfg.activation;
    a.softmax = (flags & WEKWS_FWD_SOFTMAX) ? 1 : 0;
    a.scale = m->head == WEKWS_HEAD_GLOBAL ? (float)(1.0 / (double)T) : 1.f;
    a.v_w0 = m->v_w0; a.v_b0 = m->v_b0; a.v_w1 = m->v_w1; a.v_b1 = m->v_b1;
    return cls_head_launch(a, st);
  }
  if (flags & WEKWS_FWD_SOFTMAX) {
    const long long rows = B * T;
    const int wpb = 8;
    softmax_rows_kernel<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, st>>>(d_out, rows, m->cfg.odim);
    if ((rc = check_launch("softmax_rows_kernel"))) return rc;
  }
  return WEKWS_OK;
}

// ------------------------------------------------------------------------------- training
namespace {

// The models that train on the device.  The BatchNorm models (MDTC, MDTC with a head, TCN / DS-TCN) take their
// parameters with every call on a config-only handle; FSMN and GRU train on the packed weights of a finalized handle.
enum class TrainFamily { Mdtc, MdtcHead, Tcn, Fsmn, Gru };

const char* train_label(TrainFamily f) {
  switch (f) {
    case TrainFamily::Mdtc: return "MDTC";
    case TrainFamily::MdtcHead: return "MDTC (global / last head)";
    case TrainFamily::Tcn: return "TCN / DS-TCN";
    case TrainFamily::Fsmn: return "FSMN";
    default: return "GRU";
  }
}

// A trainable model resolved from its handle: its family, the dimensions its kernels take, its parameter count
struct TrainModel {
  TrainFamily fam;
  MdtcTrainDims mdtc;                  // Mdtc, MdtcHead (odim 0: the backbone alone)
  TcnTrainDims tcn;                    // Tcn
  int n_params;                        // parameter and gradient pointers per call
};

// the dimensions of an MDTC model with the per-frame linear classifier (head == false) or with the global / last head
// (head == true: odim 0, the backbone alone), as the training kernels take them
int mdtc_dims(const wekws_model* m, const char* what, bool head, MdtcTrainDims* d) {
  const wekws_model_config& c = m->cfg;
  if (head) WEKWS_REQUIRE(c.activation == WEKWS_ACT_IDENTITY, "%s: the head trains with the Identity activation", what);
  WEKWS_REQUIRE(c.hdim == 32 || c.hdim == 64, "%s: hidden_dim %d unsupported in training (32 or 64)", what, c.hdim);
  WEKWS_REQUIRE(c.kernel_size >= 2 && c.kernel_size <= MDTC_TRAIN_MAX_K, "%s: kernel_size %d unsupported (2..%d)", what,
                c.kernel_size, MDTC_TRAIN_MAX_K);
  WEKWS_REQUIRE(c.idim >= 1 && c.idim <= MDTC_TRAIN_MAX_IDIM, "%s: input_dim %d unsupported (1..%d)", what, c.idim,
                MDTC_TRAIN_MAX_IDIM);
  const int max_odim = head ? MDTC_HEAD_TRAIN_MAX_ODIM : MDTC_TRAIN_MAX_ODIM;
  WEKWS_REQUIRE(c.odim >= 1 && c.odim <= max_odim, "%s: output_dim %d unsupported in training (1..%d)", what, c.odim,
                max_odim);
  const int L = 1 + c.num_stack * c.stack_size;
  WEKWS_REQUIRE(c.num_stack >= 1 && c.stack_size >= 1 && L <= MDTC_TRAIN_MAX_BLOCKS,
                "%s: %d stacks of %d blocks unsupported (at most %d blocks)", what, c.num_stack, c.stack_size,
                MDTC_TRAIN_MAX_BLOCKS);
  memset(d, 0, sizeof(*d));
  d->C = c.hdim; d->idim = c.idim; d->odim = head ? 0 : c.odim; d->K = c.kernel_size; d->L = L;
  d->stack_size = c.stack_size;
  d->act = c.activation == WEKWS_ACT_SIGMOID ? 1 : 0;
  d->norm_var = c.norm_var;
  int off = 0;
  for (int b = 0; b < L; ++b) {
    d->dil[b] = b == 0 ? 1 : 1 << ((b - 1) % c.stack_size);
    d->coff[b] = off;
    off += d->dil[b] * (c.kernel_size - 1);
  }
  d->pad_total = off;
  return WEKWS_OK;
}

// the dimensions of a TCN / DS-TCN model with the per-frame linear classifier, as the training kernels take them
int tcn_train_dims(const wekws_model* m, const char* what, TcnTrainDims* d) {
  const wekws_model_config& c = m->cfg;
  WEKWS_REQUIRE((c.hdim == 64 || c.hdim == 256) && c.kernel_size >= 2 && c.kernel_size <= TCN_TRAIN_MAX_K &&
                    c.num_layers >= 1 && c.num_layers <= TCN_TRAIN_MAX_LAYERS && c.idim >= 1 &&
                    c.idim <= TCN_TRAIN_MAX_IDIM && c.odim >= 1 && c.odim <= TCN_TRAIN_MAX_ODIM,
                "%s: TCN training supports hidden_dim 64 or 256, kernel_size 2..%d, 1..%d layers, input_dim <= %d and "
                "output_dim <= %d; got hidden %d, kernel %d, %d layers, input %d, output %d", what, TCN_TRAIN_MAX_K,
                TCN_TRAIN_MAX_LAYERS, TCN_TRAIN_MAX_IDIM, TCN_TRAIN_MAX_ODIM, c.hdim, c.kernel_size, c.num_layers,
                c.idim, c.odim);
  memset(d, 0, sizeof(*d));
  d->C = c.hdim; d->idim = c.idim; d->odim = c.odim; d->K = c.kernel_size; d->L = c.num_layers;
  d->ds = c.backbone == WEKWS_BACKBONE_DSTCN ? 1 : 0;
  d->act = c.activation == WEKWS_ACT_SIGMOID ? 1 : 0;
  d->norm_var = c.norm_var;
  d->pad_total = (c.kernel_size - 1) * ((1 << c.num_layers) - 1);
  return WEKWS_OK;
}

// the layer widths of an FSMN model's config (the fields the saved-activation and workspace sizes depend on)
FsmnArgs fsmn_dims(const wekws_model_config& c) {
  FsmnArgs a{};
  a.idim = c.idim; a.aff_in = c.fsmn_input_affine_dim; a.lin = c.fsmn_linear_dim; a.proj = c.fsmn_proj_dim;
  a.aff_out = c.fsmn_output_affine_dim; a.odim = c.odim; a.L = c.num_layers;
  a.lorder = c.fsmn_left_order; a.rorder = c.fsmn_right_order;
  return a;
}

// the dimensions of a GRU model's config (the fields the saved-activation and workspace sizes depend on)
GruArgs gru_dims(const wekws_model_config& c) {
  GruArgs a{};
  a.L = c.num_layers; a.H = c.hdim; a.idim = c.idim; a.odim = c.odim;
  return a;
}

// The family of a trainable model and what its calls need from the config; a TCN / DS-TCN with a head is refused.
int train_model(const wekws_model* m, const char* what, TrainModel* t) {
  WEKWS_REQUIRE(m, "%s: null handle", what);
  const int L = m->cfg.num_layers;
  int rc = WEKWS_OK;
  switch (m->cfg.backbone) {
    case WEKWS_BACKBONE_MDTC:
      t->fam = m->head == WEKWS_HEAD_LINEAR ? TrainFamily::Mdtc : TrainFamily::MdtcHead;
      if ((rc = mdtc_dims(m, what, t->fam == TrainFamily::MdtcHead, &t->mdtc))) return rc;
      t->n_params =
          t->fam == TrainFamily::Mdtc ? mdtc_train_num_params(t->mdtc.L) : mdtc_head_train_num_params(t->mdtc.L);
      return WEKWS_OK;
    case WEKWS_BACKBONE_TCN:
    case WEKWS_BACKBONE_DSTCN:
      WEKWS_REQUIRE(m->head == WEKWS_HEAD_LINEAR, "%s: the TCN model trains with the per-frame linear classifier",
                    what);
      t->fam = TrainFamily::Tcn;
      if ((rc = tcn_train_dims(m, what, &t->tcn))) return rc;
      t->n_params = tcn_train_num_params(t->tcn);
      return WEKWS_OK;
    case WEKWS_BACKBONE_FSMN:
      t->fam = TrainFamily::Fsmn;
      t->n_params = 8 + 5 * L;
      return WEKWS_OK;
    case WEKWS_BACKBONE_GRU:
      t->fam = TrainFamily::Gru;
      t->n_params = gru_num_params(L);
      return WEKWS_OK;
  }
  set_error("%s: training is not implemented for backbone %d", what, m->cfg.backbone);
  return WEKWS_ERR_INVALID;
}

bool batch_stats(TrainFamily f) { return f != TrainFamily::Fsmn && f != TrainFamily::Gru; }

// A model for wekws_train_forward / _backward and their queries: the BatchNorm models only.
int batch_stats_model(const wekws_model* m, const char* what, TrainModel* t) {
  int rc = train_model(m, what, t);
  if (rc) return rc;
  WEKWS_REQUIRE(batch_stats(t->fam), "%s: the %s model trains on the packed weights of its finalized handle, through "
                "wekws_model_load_params / wekws_model_train_forward / wekws_model_backward", what,
                train_label(t->fam));
  return WEKWS_OK;
}

// A model for wekws_model_load_params / _train_forward / _backward: FSMN (at most FSMN_MAX_TAPS memory taps) or GRU,
// finalized on the current device.
int packed_model(const wekws_model* m, const char* what, TrainModel* t) {
  int rc = train_model(m, what, t);
  if (rc) return rc;
  WEKWS_REQUIRE(!batch_stats(t->fam), "%s: the %s model takes its parameters with each call, through "
                "wekws_train_forward / wekws_train_backward", what, train_label(t->fam));
  // the backward's memory kernel keeps one register per tap; inference takes any order
  WEKWS_REQUIRE(t->fam != TrainFamily::Fsmn || m->cfg.fsmn_left_order + m->cfg.fsmn_right_order <= FSMN_MAX_TAPS,
                "%s: the FSMN model trains with at most %d memory taps (left_order + right_order), this one has "
                "%d + %d taps", what, FSMN_MAX_TAPS, m->cfg.fsmn_left_order, m->cfg.fsmn_right_order);
  if (!m->finalized) { set_error("%s called before wekws_model_finalize", what); return WEKWS_ERR_STATE; }
  WEKWS_REQUIRE(t->fam != TrainFamily::Fsmn || m->cfg.activation == WEKWS_ACT_IDENTITY,
                "%s: the FSMN model trains with the identity activation", what);
  int dev = 0;
  WEKWS_CUDA_OK(cudaGetDevice(&dev));
  WEKWS_REQUIRE(dev == m->device, "model was finalized on device %d but current device is %d", m->device, dev);
  return WEKWS_OK;
}

// The model of a wekws_train_forward / _backward call and its Dropout: n_p probabilities (MDTC 0, MDTC with a head 1,
// TCN / DS-TCN one per block), each as theta = ceil(p 2^24) in double and scale = 1 / (float)(1 - p), torch's scale.
int batch_stats_call(const wekws_model* m, const char* what, uint64_t seed, const double* h_p, int n_p, TrainModel* t,
                     MdtcHead* head, TcnDropout* drop) {
  int rc = batch_stats_model(m, what, t);
  if (rc) return rc;
  const int n_drop = t->fam == TrainFamily::Mdtc ? 0 : t->fam == TrainFamily::MdtcHead ? 1 : t->tcn.L;
  WEKWS_REQUIRE(n_p == n_drop, "%s: n_p = %d, but the %s model has %d Dropout probabilities", what, n_p,
                train_label(t->fam), n_drop);
  WEKWS_REQUIRE(n_p == 0 || h_p, "%s: null dropout probabilities", what);
  memset(head, 0, sizeof(*head));
  memset(drop, 0, sizeof(*drop));
  head->last = m->head == WEKWS_HEAD_LAST ? 1 : 0;
  head->odim = m->cfg.odim;
  head->seed = drop->seed = seed;
  uint32_t* theta = t->fam == TrainFamily::MdtcHead ? &head->theta : drop->theta;
  float* scale = t->fam == TrainFamily::MdtcHead ? &head->scale : drop->scale;
  for (int l = 0; l < n_p; ++l) {
    WEKWS_REQUIRE(h_p[l] >= 0.0 && h_p[l] <= 1.0, "%s: dropout probability %g (number %d) is outside [0, 1]", what,
                  h_p[l], l);
    theta[l] = (uint32_t)ceil(h_p[l] * 16777216.0);
    scale[l] = 1.0f / (float)(1.0 - h_p[l]);
  }
  return WEKWS_OK;
}

int num_batch_norms(const TrainModel& t) { return t.fam == TrainFamily::Tcn ? tcn_train_num_bns(t.tcn) : 3 * t.mdtc.L; }

// The arguments of a batch-statistics training forward of a model of width C and output width odim with nbn
// BatchNorms.
int batch_stats_forward_check(const char* what, int64_t B, int64_t T, int C, int odim, int n, int n_expected, int nbn,
                              const float* d_feats, const float* const* h_params, const float* d_cmvn_mean,
                              const float* d_cmvn_istd, float* const* h_running, const double* h_bn,
                              const float* d_out, const float* d_out_cache, const float* d_saved, int save,
                              const void* d_workspace) {
  WEKWS_REQUIRE(B >= 1 && T >= 1 && B * T >= 2 && B * T * C < (1LL << 31) && B * T * odim < (1LL << 31),
                "%s: B = %lld, T = %lld unsupported (B * T >= 2 frames are needed for batch statistics)", what,
                (long long)B, (long long)T);
  WEKWS_REQUIRE(n == n_expected, "%s: expected %d parameters, got %d", what, n_expected, n);
  WEKWS_REQUIRE(d_feats && h_params && h_running && h_bn && d_out && d_out_cache && d_workspace && (!save || d_saved),
                "%s: null argument", what);
  WEKWS_REQUIRE((d_cmvn_mean == nullptr) == (d_cmvn_istd == nullptr), "%s: pass both CMVN buffers or neither", what);
  for (int i = 0; i < n; ++i) WEKWS_REQUIRE(h_params[i] != nullptr, "%s: parameter %d is null", what, i);
  for (int i = 0; i < 2 * nbn; ++i) WEKWS_REQUIRE(h_running[i] != nullptr, "%s: running statistic %d is null", what, i);
  for (int i = 0; i < nbn; ++i)
    WEKWS_REQUIRE(h_bn[2 * i] >= 0.0 && h_bn[2 * i] <= 1.0 && h_bn[2 * i + 1] > 0.0,
                  "%s: BatchNorm %d has momentum %g, eps %g", what, i, h_bn[2 * i], h_bn[2 * i + 1]);
  return WEKWS_OK;
}

// The arguments of its backward; args_present: every pointer argument but the parameters and gradients is non-null.
int batch_stats_backward_check(const char* what, int64_t B, int64_t T, int C, int odim, int n, int n_expected,
                               const float* const* h_params, float* const* h_grads, bool args_present) {
  WEKWS_REQUIRE(B >= 1 && T >= 1 && B * T >= 2 && B * T * C < (1LL << 31) && B * T * odim < (1LL << 31),
                "%s: bad B/T", what);
  WEKWS_REQUIRE(n == n_expected, "%s: expected %d parameters, got %d", what, n_expected, n);
  WEKWS_REQUIRE(args_present && h_params && h_grads, "%s: null argument", what);
  for (int i = 0; i < n; ++i)
    WEKWS_REQUIRE(h_params[i] != nullptr && h_grads[i] != nullptr, "%s: parameter or gradient %d is null", what, i);
  return WEKWS_OK;
}

}  // namespace

extern "C" int wekws_train_num_params(const wekws_model* m) {
  TrainModel t;
  return train_model(m, "wekws_train_num_params", &t) ? 0 : t.n_params;
}

extern "C" int64_t wekws_train_saved_floats(const wekws_model* m, int64_t B, int64_t T) {
  const char* what = "wekws_train_saved_floats";
  TrainModel t;
  int rc = train_model(m, what, &t);
  if (rc) return rc;
  WEKWS_REQUIRE(B >= 0 && T >= 0, "%s: B, T >= 0 are required", what);
  switch (t.fam) {
    case TrainFamily::Mdtc: return mdtc_train_saved_floats(t.mdtc, B * T);
    case TrainFamily::MdtcHead: return mdtc_head_train_saved_floats(t.mdtc, B, T);
    case TrainFamily::Tcn: return tcn_train_saved_floats(t.tcn, B * T);
    case TrainFamily::Fsmn: return B * T * fsmn_saved_per_frame(fsmn_dims(m->cfg));
    default: return B * T * gru_saved_per_frame(m->cfg.num_layers, m->cfg.hdim);
  }
}

extern "C" int64_t wekws_train_backward_workspace_bytes(const wekws_model* m, int64_t B, int64_t T) {
  const char* what = "wekws_train_backward_workspace_bytes";
  TrainModel t;
  int rc = train_model(m, what, &t);
  if (rc) return rc;
  WEKWS_REQUIRE(B >= 0 && T >= 0, "%s: B, T >= 0 are required", what);
  switch (t.fam) {
    case TrainFamily::Mdtc: return mdtc_backward_workspace_bytes(t.mdtc, B * T);
    case TrainFamily::MdtcHead: return mdtc_head_backward_workspace_bytes(t.mdtc, B, T);
    case TrainFamily::Tcn: return tcn_backward_workspace_bytes(t.tcn, B * T);
    case TrainFamily::Fsmn: return (int64_t)sizeof(float) * fsmn_backward_workspace_floats(fsmn_dims(m->cfg), B * T);
    default: return (int64_t)sizeof(float) * gru_backward_workspace_floats(gru_dims(m->cfg), B * T);
  }
}

extern "C" int wekws_train_backward_launches(const wekws_model* m) {
  TrainModel t;
  if (train_model(m, "wekws_train_backward_launches", &t)) return 0;
  switch (t.fam) {
    case TrainFamily::Mdtc: return mdtc_train_backward_launches(t.mdtc.L);
    case TrainFamily::MdtcHead: return mdtc_head_backward_launches(t.mdtc.L);
    case TrainFamily::Tcn: return tcn_train_backward_launches(t.tcn);
    case TrainFamily::Fsmn: return fsmn_backward_launches(m->cfg.num_layers);
    default: return gru_backward_launches(m->cfg.num_layers);
  }
}

extern "C" int64_t wekws_train_workspace_bytes(const wekws_model* m, int64_t B, int64_t T, int save) {
  const char* what = "wekws_train_workspace_bytes";
  TrainModel t;
  int rc = batch_stats_model(m, what, &t);
  if (rc) return rc;
  WEKWS_REQUIRE(B >= 0 && T >= 0, "%s: B, T >= 0 are required", what);
  switch (t.fam) {
    case TrainFamily::Mdtc: return mdtc_train_workspace_bytes(t.mdtc, B * T, save != 0);
    case TrainFamily::MdtcHead: return mdtc_head_train_workspace_bytes(t.mdtc, B, T, save != 0);
    default: return tcn_train_workspace_bytes(t.tcn, B * T, save != 0);
  }
}

extern "C" int wekws_train_forward_launches(const wekws_model* m) {
  TrainModel t;
  if (batch_stats_model(m, "wekws_train_forward_launches", &t)) return 0;
  switch (t.fam) {
    case TrainFamily::Mdtc: return mdtc_train_forward_launches(t.mdtc.L);
    case TrainFamily::MdtcHead: return mdtc_head_train_forward_launches(t.mdtc.L);
    default: return tcn_train_forward_launches(t.tcn);
  }
}

extern "C" int wekws_train_forward(const wekws_model* m, const float* d_feats, const float* const* h_params, int n,
                                   const float* d_cmvn_mean, const float* d_cmvn_istd, float* const* h_running,
                                   const double* h_bn, uint64_t seed, const double* h_p, int n_p, float* d_out,
                                   float* d_out_cache, float* d_saved, int save, void* d_workspace, int64_t B,
                                   int64_t T, void* stream) {
  const char* what = "wekws_train_forward";
  TrainModel t;
  MdtcHead head;
  TcnDropout drop;
  int rc = batch_stats_call(m, what, seed, h_p, n_p, &t, &head, &drop);
  if (rc) return rc;
  if ((rc = batch_stats_forward_check(what, B, T, m->cfg.hdim, m->cfg.odim, n, t.n_params, num_batch_norms(t), d_feats,
                                      h_params, d_cmvn_mean, d_cmvn_istd, h_running, h_bn, d_out, d_out_cache, d_saved,
                                      save, d_workspace)))
    return rc;
  float* saved = save ? d_saved : nullptr;
  cudaStream_t st = (cudaStream_t)stream;
  switch (t.fam) {
    case TrainFamily::Mdtc:
      return mdtc_train_forward_launch(t.mdtc, d_feats, h_params, d_cmvn_mean, d_cmvn_istd, h_running, h_bn, d_out,
                                       d_out_cache, saved, d_workspace, (int)B, (int)T, st);
    case TrainFamily::MdtcHead:
      return mdtc_head_train_forward_launch(t.mdtc, head, d_feats, h_params, d_cmvn_mean, d_cmvn_istd, h_running, h_bn,
                                            d_out, d_out_cache, saved, d_workspace, (int)B, (int)T, st);
    default:
      return tcn_train_forward_launch(t.tcn, drop, d_feats, h_params, d_cmvn_mean, d_cmvn_istd, h_running, h_bn, d_out,
                                      d_out_cache, saved, d_workspace, (int)B, (int)T, st);
  }
}

extern "C" int wekws_train_backward(const wekws_model* m, const float* d_feats, const float* const* h_params, int n,
                                    const float* d_cmvn_mean, const float* d_cmvn_istd, const float* d_saved,
                                    const float* d_out, const float* d_grad_out, uint64_t seed, const double* h_p,
                                    int n_p, int64_t B, int64_t T, float* const* h_grads, void* d_workspace,
                                    void* stream) {
  const char* what = "wekws_train_backward";
  TrainModel t;
  MdtcHead head;
  TcnDropout drop;
  int rc = batch_stats_call(m, what, seed, h_p, n_p, &t, &head, &drop);
  if (rc) return rc;
  const bool reads_out = t.fam == TrainFamily::Tcn;      // only the TCN backward reads the logits
  if ((rc = batch_stats_backward_check(what, B, T, m->cfg.hdim, m->cfg.odim, n, t.n_params, h_params, h_grads,
                                       d_feats && d_saved && (d_out || !reads_out) && d_grad_out && d_workspace)))
    return rc;
  cudaStream_t st = (cudaStream_t)stream;
  switch (t.fam) {
    case TrainFamily::Mdtc:
      return mdtc_backward_launch(t.mdtc, d_feats, h_params, d_cmvn_mean, d_cmvn_istd, d_saved, d_grad_out, (int)B,
                                  (int)T, h_grads, d_workspace, st);
    case TrainFamily::MdtcHead:
      return mdtc_head_backward_launch(t.mdtc, head, d_feats, h_params, d_cmvn_mean, d_cmvn_istd, d_saved, d_grad_out,
                                       (int)B, (int)T, h_grads, d_workspace, st);
    default:
      return tcn_backward_launch(t.tcn, drop, d_feats, h_params, d_cmvn_mean, d_cmvn_istd, d_saved, d_out, d_grad_out,
                                 (int)B, (int)T, h_grads, d_workspace, st);
  }
}

extern "C" int wekws_model_load_params(wekws_model* m, const float* const* h_params, int n, void* stream) {
  const char* what = "wekws_model_load_params";
  TrainModel t;
  int rc = packed_model(m, what, &t);
  if (rc) return rc;
  WEKWS_REQUIRE(h_params && n == t.n_params, "%s: expected the %d parameters of a %d-layer %s model, got %d", what,
                t.n_params, m->cfg.num_layers, train_label(t.fam), n);
  if (m->params.size() != (size_t)n) {
    set_error("internal: %s: the pack holds %zu parameters, not %d", what, m->params.size(), n);
    return WEKWS_ERR_INVALID;
  }
  FsmnPackArgs p{};
  p.packed = m->d_vec;
  p.n = n;
  for (int i = 0; i < n; ++i) {
    WEKWS_REQUIRE(h_params[i] != nullptr, "%s: parameter %d is null", what, i);
    const PackedParam& e = m->params[i];
    p.p[i] = {h_params[i], e.dst, e.rows, e.cols, e.ld};
  }
  return fsmn_pack_launch(p, (cudaStream_t)stream);
}

extern "C" int wekws_model_train_forward(wekws_model* m, const float* d_feats, float* d_out, float* d_out_cache,
                                         float* d_saved, int64_t B, int64_t T, void* stream) {
  const char* what = "wekws_model_train_forward";
  TrainModel t;
  int rc = packed_model(m, what, &t);
  if (rc) return rc;
  WEKWS_REQUIRE(B >= 1 && T >= 1 && B < (1 << 30) && T < (1 << 30), "%s: bad B/T", what);
  WEKWS_REQUIRE(d_feats && d_out && d_out_cache && d_saved, "%s: null tensor", what);
  cudaStream_t st = (cudaStream_t)stream;
  if (t.fam == TrainFamily::Gru) {
    GruArgs a = m->gru;                        // the FP32 kernel whatever the precision mode
    a.feats = d_feats; a.in_cache = nullptr; a.out = d_out; a.out_cache = d_out_cache;
    a.B = (int)B; a.T = (int)T; a.saved = d_saved;
    return gru_launch(a, st, true);
  }
  // FSMN: the time chunks of wekws_model_forward, each launch also storing its frames' activations
  const int maxT = fsmn_tile_rows();
  const int nchunk = (int)((T + maxT - 1) / maxT);
  const int Tc = (int)((T + nchunk - 1) / nchunk);
  for (int64_t t0 = 0; t0 < T; t0 += Tc) {
    FsmnArgs a = m->fsmn;
    a.feats = d_feats + t0 * m->cfg.idim;
    a.out = d_out + t0 * m->cfg.odim;
    a.in_cache = t0 == 0 ? nullptr : d_out_cache;
    a.out_cache = d_out_cache;
    a.B = (int)B;
    a.T = (int)(T - t0 < Tc ? T - t0 : Tc);
    a.feat_bstride = T * m->cfg.idim;
    a.out_bstride = T * m->cfg.odim;
    a.saved = d_saved; a.save_T = (int)T; a.save_t0 = (int)t0;
    if ((rc = fsmn_train_launch(a, st))) return rc;
  }
  return WEKWS_OK;
}

extern "C" int wekws_model_backward(wekws_model* m, const float* d_feats, const float* d_saved, const float* d_out,
                                    const float* d_grad_out, int64_t B, int64_t T, float* const* h_grads, int n,
                                    void* d_workspace, void* stream) {
  const char* what = "wekws_model_backward";
  TrainModel t;
  int rc = packed_model(m, what, &t);
  if (rc) return rc;
  const bool gru = t.fam == TrainFamily::Gru;              // only the GRU backward reads the logits
  WEKWS_REQUIRE(B >= 1 && T >= 1 && B < (1 << 30) && T < (1 << 30), "%s: bad B/T", what);
  WEKWS_REQUIRE(d_feats && d_saved && (d_out || !gru) && d_grad_out && d_workspace && h_grads, "%s: null argument",
                what);
  WEKWS_REQUIRE(n == t.n_params, "%s: expected %d gradient buffers, got %d", what, t.n_params, n);
  for (int i = 0; i < n; ++i) WEKWS_REQUIRE(h_grads[i] != nullptr, "%s: gradient buffer %d is null", what, i);
  cudaStream_t st = (cudaStream_t)stream;
  if (gru)
    return gru_backward_launch(m->gru, d_feats, d_saved, d_out, d_grad_out, (int)B, (int)T, h_grads,
                               (float*)d_workspace, st);
  return fsmn_backward_launch(m->fsmn, d_feats, d_saved, d_grad_out, (int)B, (int)T, h_grads, (float*)d_workspace, st);
}

extern "C" int wekws_dropout_mask(uint64_t seed, int64_t B, int64_t T, int64_t C, int layer, uint32_t theta,
                                  uint8_t* d_out, void* stream) {
  WEKWS_REQUIRE(B >= 0 && T >= 0 && C >= 0 && B < (1LL << 31) && T < (1LL << 31) && C < (1LL << 31) && layer >= 0 &&
                    theta <= (1u << 24), "wekws_dropout_mask: bad arguments");
  WEKWS_REQUIRE(B * T * C == 0 || d_out, "wekws_dropout_mask: null output");
  return dropout_mask_launch(seed, B, T, (int)C, layer, theta, d_out, (cudaStream_t)stream);
}

extern "C" int wekws_pipeline_forward(wekws_fbank* fb, wekws_model* m, const void* d_pcm, int pcm_dtype,
                                      int64_t B, int64_t num_samples, int64_t pcm_stride,
                                      float* d_feat_scratch, const float* d_in_cache, float* d_out,
                                      float* d_out_cache, uint32_t flags, void* stream) {
  WEKWS_REQUIRE(fb && m && d_feat_scratch, "wekws_pipeline_forward: null argument");
  WEKWS_REQUIRE(wekws_fbank_feature_dim(fb) == m->cfg.idim, "pipeline: the front-end produces %d features but the model expects input_dim %d",
                wekws_fbank_feature_dim(fb), m->cfg.idim);
  const int64_t frames = wekws_fbank_num_frames(fb, num_samples);
  // The feature tensor only lives between the two launches.  Pin it in L2 for their duration (persisting access-policy
  // window on this stream): the front-end's writes stay in the cache, the model kernel's first-Linear reads hit there,
  // and the lines are released (not written back as "persisting") afterwards -- the 320 B/frame never has to make the
  // HBM round trip as long as B * frames * idim * 4 fits the device's persisting-L2 carve-out.
  cudaStream_t st = (cudaStream_t)stream;
  const size_t feat_bytes = (size_t)B * (size_t)frames * (size_t)m->cfg.idim * sizeof(float);
  bool windowed = false;
  if (feat_bytes > 0) {
    int dev = 0, max_persist = 0, max_window = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev) == cudaSuccess && max_persist > 0) {
      static bool limit_set[64] = {false};
      if (dev >= 0 && dev < 64 && !limit_set[dev]) {
        cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, (size_t)max_persist);
        limit_set[dev] = true;
      }
      cudaStreamAttrValue attr;
      memset(&attr, 0, sizeof(attr));
      attr.accessPolicyWindow.base_ptr = d_feat_scratch;
      attr.accessPolicyWindow.num_bytes = feat_bytes < (size_t)max_window ? feat_bytes : (size_t)max_window;
      attr.accessPolicyWindow.hitRatio = feat_bytes <= (size_t)max_persist ? 1.0f : (float)max_persist / (float)feat_bytes;
      attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
      attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
      windowed = cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &attr) == cudaSuccess;
    }
    cudaGetLastError();      // the window is an optimisation: never fatal
  }
  int rc = wekws_fbank_forward(fb, d_pcm, pcm_dtype, B, num_samples, pcm_stride, nullptr, nullptr, nullptr,
                               d_feat_scratch, frames, stream);
  if (rc == 0) rc = wekws_model_forward(m, d_feat_scratch, d_in_cache, d_out, d_out_cache, B, frames, flags, stream);
  if (windowed) {
    cudaStreamAttrValue attr;
    memset(&attr, 0, sizeof(attr));
    attr.accessPolicyWindow.num_bytes = 0;                       // window off for whatever the caller runs next
    cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &attr);
    cudaGetLastError();
  }
  return rc;
}
