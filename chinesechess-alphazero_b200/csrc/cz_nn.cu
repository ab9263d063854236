// cz_nn.cu — policy + value network forward (agent/model.py:32-83) on H100 (sm_90a).
//
//   packed boards --k_conv_first--> activations [B*90][C] (5x5 input conv over one-hot planes is a gather-sum
//                                   of <= 25 weight rows per pixel; plane encoding never materialises)
//   2 x blocks of  igemm::k_igemm   3x3 conv as implicit GEMM on wgmma (BN folded, +skip, ReLU fused)
//   k_heads                         1x1 policy/value convs + BN + ReLU, value MLP + tanh
//   igemm::k_igemm (GEMM mode)      policy_out Dense 360 -> 2086 on wgmma
//   k_softmax                       2086-way softmax
//
// BatchNormalization is inference-mode (moving statistics, eps = 1e-3, data/model/model_best_config.json)
// and folded into fp16 weights + fp32 shift.  Weights arrive in Keras layout, caller-owned.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <utility>
#include <vector>

#include "cz_err.h"
#include "cz_igemm.cuh"
#include "cz_nn.cuh"
#include "cz_nn_host.cuh"

namespace cznn {

constexpr int kLabels = CZ_N_LABELS;
// Head widths are a property of the weight file: agent/model.py:47-61 builds 4 policy / 2 value channels, the older configs shipped
// under data/model/ (model_128f.json, model_256f.json: 2 / 4; model_128_l1_config.json: 32 / 4) are served too.
//   pol_k1 = policy features (policy channels x 90) padded to whole 64-column k-blocks, pol_k = 3 * pol_k1:
//            the policy Dense runs as a split-precision GEMM on the tensor cores:
                                   //   x = x_hi + x_lo, w = w_hi + w_lo (fp16 each); logits = x_hi.w_hi + x_lo.w_hi + x_hi.w_lo
                                   // laid out along K as A' = [x_hi | x_lo | x_hi], W' = [w_hi | w_hi | w_lo] -> one GEMM, ~fp32 accuracy
                                   // (fp16 operands alone cost 1.1e-3 of policy probability on the reference's trained 192x10 net)
constexpr int kPolN = 2304;     // 2086 labels padded to 9 N tiles of 256
constexpr float kBnEps = 1e-3f;

// ------------------------------------------------------------------------------------------------
// driver entry point for tensor-map encoding (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;
static EncodeIm2colFn g_encode_im2col = nullptr;

static int load_encode() {
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || !fn) return cz_fail(CZ_ERR_CUDA, "cuTensorMapEncodeTiled not available: %s", cudaGetErrorString(e));
  g_encode = (EncodeTiledFn)fn;
  fn = nullptr;
  e = cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qres);
  if (e == cudaSuccess && fn) g_encode_im2col = (EncodeIm2colFn)fn;
  return 0;
}

// fp16 NHWC activations [n][10][9][c] read in im2col mode for a 3x3 "same" convolution: the bounding box of base pixels is
// [-1, dim-2] in w and h (lower corner = -pad, upper corner = pad - (filter-1)), 64 channels x `pixels` output pixels per load;
// taps outside the image are zero-filled by the TMA unit, and the pixel column walks across rows and images.
int make_map_im2col(CUtensorMap* m, const void* base, int c, long long n_images, int pixels) {
  if (load_encode()) return CZ_ERR_CUDA;
  if (!g_encode_im2col) return cz_fail(CZ_ERR_UNSUPPORTED, "cuTensorMapEncodeIm2col not available");
  cuuint64_t dims[4] = {(cuuint64_t)c, 9, 10, (cuuint64_t)n_images};
  cuuint64_t strides[3] = {(cuuint64_t)c * 2, (cuuint64_t)c * 2 * 9, (cuuint64_t)c * 2 * 90};
  int lower[2] = {-1, -1}, upper[2] = {-1, -1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = g_encode_im2col(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, lower, upper, 64, (cuuint32_t)pixels,
                               es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cz_fail(CZ_ERR_CUDA, "cuTensorMapEncodeIm2col failed: %d", (int)r);
  return 0;
}

// fp16 matrix [rows][k] (k contiguous), box {64, rows_per_box}
int make_map_2d(CUtensorMap* m, const void* base, int k, long long rows, int rows_per_box) {
  if (load_encode()) return CZ_ERR_CUDA;
  cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)k * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)rows_per_box};
  cuuint32_t es[2] = {1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cz_fail(CZ_ERR_CUDA, "cuTensorMapEncodeTiled(2d) failed: %d", (int)r);
  return 0;
}

// fp16 matrix [rows][cols] as the staged conv epilogue stores it: boxes of 32 columns x 64 rows, 64-byte rows in shared memory
static int make_map_epi(CUtensorMap* m, const void* base, int cols, long long rows) {
  if (load_encode()) return CZ_ERR_CUDA;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)igemm::kEpiCols, 64};
  cuuint32_t es[2] = {1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cz_fail(CZ_ERR_CUDA, "cuTensorMapEncodeTiled(epilogue) failed: %d", (int)r);
  return 0;
}

static int g_num_sms = 0;
int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

// Programmatic dependent launch: a conv's CTAs may become resident and run their prologue (barrier init, tensor-map prefetch)
// while the previous kernel of the stream is still running; griddepcontrol.wait in the kernel orders the data.
template <int N_TILE, int M_TILE, bool CONV>
static int launch_igemm_t(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmOut, const igemm::Args& a, cudaStream_t st) {
  using C = igemm::Cfg<N_TILE, M_TILE, CONV>;
  static bool attr_set = false;
  if (!attr_set) {
    CZ_CUDA(cudaFuncSetAttribute(igemm::k_igemm<N_TILE, M_TILE, CONV>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes));
    attr_set = true;
  }
  const int tiles = a.m_tiles * a.n_tiles;
  if (tiles <= 0) return 0;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  cudaLaunchConfig_t lc;
  memset(&lc, 0, sizeof(lc));
  lc.gridDim = dim3(grid); lc.blockDim = dim3(igemm::kThreads); lc.dynamicSmemBytes = C::kSmemBytes; lc.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = at; lc.numAttrs = 1;
  CZ_CUDA(cudaLaunchKernelEx(&lc, igemm::k_igemm<N_TILE, M_TILE, CONV>, tmA, tmB, tmOut, a));
  CZ_CUDA(cudaGetLastError());
  return 0;
}
// With `out_map` (make_map_epi of a.out) the full M tiles of a conv that has fp16 output only and no skip stream leave
// through the staged epilogue.
int launch_igemm(int n_tile, const CUtensorMap& tmA, const CUtensorMap& tmB, const igemm::Args& a0, cudaStream_t st, const CUtensorMap* out_map) {
  igemm::Args a = a0;
  a.staged = out_map && a.conv && !a.out_f32 && !a.residual && !a.residual32 && !a.out32;
  const CUtensorMap& tmOut = a.staged ? *out_map : tmA;    // not used unless staged
  if (a.conv) {
    const int key = n_tile * 1000 + a.tile_m;
    switch (key) {                                          // the tiles conv_args chooses
      case 64128: return launch_igemm_t<64, 128, true>(tmA, tmB, tmOut, a, st);
      case 64256: return launch_igemm_t<64, 256, true>(tmA, tmB, tmOut, a, st);
      case 128128: return launch_igemm_t<128, 128, true>(tmA, tmB, tmOut, a, st);
      case 128256: return launch_igemm_t<128, 256, true>(tmA, tmB, tmOut, a, st);
      case 192128: return launch_igemm_t<192, 128, true>(tmA, tmB, tmOut, a, st);
    }
    return cz_fail(CZ_ERR_UNSUPPORTED, "igemm: unsupported conv tile %d x %d", a.tile_m, n_tile);
  }
  switch (n_tile) {
    case 64: return launch_igemm_t<64, igemm::kTileM, false>(tmA, tmB, tmOut, a, st);
    case 128: return launch_igemm_t<128, igemm::kTileM, false>(tmA, tmB, tmOut, a, st);
    case 192: return launch_igemm_t<192, igemm::kTileM, false>(tmA, tmB, tmOut, a, st);
    case 256: return launch_igemm_t<256, igemm::kTileM, false>(tmA, tmB, tmOut, a, st);
  }
  return cz_fail(CZ_ERR_UNSUPPORTED, "igemm: unsupported N tile %d (filters must be 64/128/192/256)", n_tile);
}
// Small batches (one game's leaves: the UCI / play_games latency path): 64-column tiles, m_tiles x C/64 work items, as long as
// they fit one wave of CTAs.  The weight map then has 64-row boxes (NetWeights::map_w_64).
static bool use_n_split(int n_boards, int c) {
  if (c <= 64) return false;
  const int m_tiles = (n_boards * 90 + igemm::kTileM - 1) / igemm::kTileM;
  return m_tiles * (c / 64) <= num_sms();
}
// Conv tiles: N = 128 at C = 256 (two N tiles), C itself below; the small-batch form is 128 x 64.  M = 256 pixels (two m64
// blocks per consumer warpgroup, 128 accumulators per thread at N = 128) halves the weight bytes each CTA loads per output
// pixel, as long as the 256-pixel tiles fill at least 8 waves of CTAs: with fewer, the last, partly filled wave costs more
// than the bytes save (c2, at most 2048 positions at 128x7, makes 720 such tiles, 5.5 waves, and ran 2.5 % slower with them on
// an H100).  C = 192 stays
// at 128 pixels: 2 x m64n192 would need 192 accumulators.
int conv_tile_n(int c, bool split) { return split ? 64 : c == 256 ? 128 : c; }
static int conv_tile_m(int n_boards, int c, bool split) {
  if (split || c == 192) return 128;
  const long long tiles = ((long long)n_boards * 90 + 255) / 256 * (c / conv_tile_n(c, false));
  return tiles >= 8LL * num_sms() ? 256 : 128;
}
igemm::Args conv_args(int n_boards, int c, const float* bias, const __half* residual, void* out, int relu, bool split) {
  igemm::Args a;
  memset(&a, 0, sizeof(a));
  a.n_taps = 9; a.k_chunks = c / 64;
  a.tile_m = conv_tile_m(n_boards, c, split);
  a.rows = n_boards * 90; a.m_tiles = (a.rows + a.tile_m - 1) / a.tile_m; a.n_tiles = c / conv_tile_n(c, split);
  a.n_total = c; a.n_valid = c; a.ldo = c; a.conv = 1; a.relu = relu; a.out_f32 = 0;
  a.bias = bias; a.residual = residual; a.out = out; a.rows_per_unit = 90;
  return a;
}

static igemm::Args dense_args(int m, int n_valid, int n_pad, int k_pad, int n_tile, const float* bias, float* out, int ldo) {
  igemm::Args a;
  memset(&a, 0, sizeof(a));
  a.n_taps = 1; a.k_chunks = k_pad / 64;
  a.tile_m = igemm::kTileM; a.rows = m; a.m_tiles = (m + igemm::kTileM - 1) / igemm::kTileM; a.n_tiles = n_pad / n_tile;
  a.n_total = n_pad; a.n_valid = n_valid; a.ldo = ldo; a.conv = 0; a.relu = 0; a.out_f32 = 1;
  a.bias = bias; a.residual = nullptr; a.out = out;
  return a;
}

// ------------------------------------------------------------------------------------------------
// small kernels
// packed board -> plane index per network pixel (pix = r*9 + col, r = 9 - y), -1 = empty
__device__ __forceinline__ int plane_of(uint8_t c) { return c == 0 ? -1 : ((c & 8) ? c - 2 : c - 1); }

// 5x5 "same" input convolution + BN + ReLU from packed boards (model.py:34-41, static_env.py:137-156 fused).
// The 14 input planes are one-hot, so an output pixel is the sum of <= 25 weight rows w[tap][plane(piece on the
// tapped square)][:].  Phase 1: 90 threads list the occupied taps of their pixel (row index = tap*14 + plane);
// phase 2: every thread owns two adjacent output channels of a subset of the pixels and walks their lists (half2 loads, fp32
// accumulate).  grid = batch, block = (C/2) * n_groups >= 96 threads (conv_first_threads).  w: HWIO [5][5][in_planes][C] fp16 (BN scale folded).
// in_planes = 28 (use_history, static_env.py:158-194): every board record is followed by the history board whose pieces
// select planes 14-27; board_stride = bytes between records.
__global__ void k_conv_first(const uint8_t* __restrict__ boards, const __half* __restrict__ w,
                             const float* __restrict__ shift, __half* __restrict__ out, float* __restrict__ out32, int c_out,
                             int in_planes, int board_stride, const int* __restrict__ n_dev) {
  if ((int)blockIdx.x >= __ldg(n_dev)) return;              // fixed-shape launch: the batch size lives on the device
  __shared__ int8_t pl[2][90];
  __shared__ uint16_t rows[90][52];
  __shared__ uint8_t cnt[90];
  const int b = blockIdx.x, t = threadIdx.x;
  const int n_boards = in_planes / 14;
  if (t < 90) {
    const int r = t / 9, col = t % 9;
    for (int h = 0; h < n_boards; ++h)
      pl[h][t] = (int8_t)plane_of(boards[(size_t)b * board_stride + h * CZ_BOARD_STRIDE + (9 - r) * 9 + col]);
  }
  __syncthreads();
  // gridDim.y slices of the 90 pixels (small batches: one CTA per position would leave the GPU to a handful of CTAs that each
  // walk 90 x <= 50 dependent-latency loads)
  const int per = (90 + (int)gridDim.y - 1) / (int)gridDim.y, p0 = (int)blockIdx.y * per, p1 = p0 + per < 90 ? p0 + per : 90;
  if (t < p1 - p0) {
    const int r = (p0 + t) / 9, col = (p0 + t) % 9;
    int n = 0;
    for (int kh = 0; kh < 5; ++kh) {
      const int rr = r + kh - 2;
      if (rr < 0 || rr > 9) continue;
      for (int kw = 0; kw < 5; ++kw) {
        const int cc = col + kw - 2;
        if (cc < 0 || cc > 8) continue;
        for (int h = 0; h < n_boards; ++h) {
          const int p = pl[h][rr * 9 + cc];
          if (p >= 0) rows[t][n++] = (uint16_t)((kh * 5 + kw) * in_planes + h * 14 + p);
        }
      }
    }
    cnt[t] = (uint8_t)n;
  }
  __syncthreads();
  // phase 2: thread = (channel pair, pixel group): blockDim.x = (c_out / 2) * n_groups, group g takes pixels g, g + n_groups, ...
  const int pairs = c_out / 2;
  const int c = 2 * (t % pairs), grp = t / pairs, n_groups = blockDim.x / pairs;
  if (grp >= n_groups) return;
  const float2 sh = *reinterpret_cast<const float2*>(shift + c);
  __half* o = out + (size_t)b * 90 * c_out;
  const __half2* w2 = reinterpret_cast<const __half2*>(w + c);
  const int stride2 = c_out / 2;
  for (int pix = p0 + grp; pix < p1; pix += n_groups) {
    float a0 = sh.x, a1 = sh.y;
    const int n = cnt[pix - p0];
    for (int k = 0; k < n; ++k) {
      const float2 v = __half22float2(__ldg(w2 + (size_t)rows[pix - p0][k] * stride2));
      a0 += v.x; a1 += v.y;
    }
    a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f);
    *reinterpret_cast<__half2*>(o + (size_t)pix * c_out + c) = __floats2half2_rn(a0, a1);
    if (out32) *reinterpret_cast<float2*>(out32 + ((size_t)b * 90 + pix) * c_out + c) = make_float2(a0, a1);
  }
}

// one-hot planes [B][in_planes][10][9] f32 -> packed boards (inverse of state_to_planes / state_history_to_planes):
// in_planes / 14 consecutive board records per position
__global__ void k_planes_to_boards(const float* __restrict__ planes, uint8_t* __restrict__ boards, int n, int in_planes) {
  const int b = blockIdx.x;
  if (b >= n) return;
  const int t = threadIdx.x;
  if (t < 96) {
    for (int h = 0; h < in_planes / 14; ++h) {
      uint8_t code = 0;
      if (t < 90) {
        const int y = t / 9, x = t % 9, r = 9 - y;
        for (int p = 0; p < 14; ++p)
          if (planes[((size_t)b * in_planes + h * 14 + p) * 90 + r * 9 + x] > 0.5f) code = (uint8_t)(p < 7 ? p + 1 : p + 2);
      }
      boards[((size_t)b * (in_planes / 14) + h) * CZ_BOARD_STRIDE + t] = code;
    }
  }
}

// Heads (model.py:47-63): 1x1 conv to 4 policy + 2 value channels, BN, ReLU; policy features to the GEMM
// operand [B][384] (index c*90 + pix, Keras Flatten of channels_first); value: Dense(H)+ReLU, Dense(1)+tanh.
// A block handles kHeadPos positions so the 180 x H value weights are read once per group.
// Phase 1: one thread per (position, pixel): it streams that pixel's C activations (16-byte loads along its own row; the rows
// of a warp's 32 pixels are adjacent in memory) against the 6 x C folded weights held in shared memory (broadcast reads) —
// no cross-lane reduction.  (The round-1 version reduced six sums with 30 shuffles per pixel: 110 us per 2048 positions.)
constexpr int kHeadPos = 4;
constexpr int kMaxHeadOut = 36;                                   // 32 policy + 4 value channels
static size_t heads_smem_bytes(int c_in, int n_out) { return ((size_t)kHeadPos * n_out * 90 + (size_t)(c_in / 8) * n_out * 8 + kHeadPos * 8) * sizeof(float); }
__global__ void __launch_bounds__(256) k_heads(const __half* __restrict__ act, const float* __restrict__ act32, int c_in,
                                                const int* __restrict__ n_dev, int pol_c, int val_c, int pol_k1,
                                                const float* __restrict__ wh,      // [pol_c + val_c][c_in], BN scale folded
                                                const float* __restrict__ shifth,  // [pol_c + val_c]
                                                const float* __restrict__ wv1,     // [val_c * 90][H]
                                                const float* __restrict__ bv1,     // [H]
                                                const float* __restrict__ wv2,     // [H]
                                                const float* __restrict__ bv2,     // [1]
                                                int hidden, __half* __restrict__ pol_feat, float* __restrict__ value,
                                                int hp) {          // positions per block: kHeadPos, or 1 for small batches
  extern __shared__ __align__(16) float hsm[];
  const int n_out = pol_c + val_c;
  float* feat = hsm;                                         // [kHeadPos][n_out][90]
  float* wsm = feat + kHeadPos * n_out * 90;                 // [c_in / 8][n_out][8]
  float* red = wsm + (c_in / 8) * n_out * 8;                 // [kHeadPos][8]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b0 = blockIdx.x * hp;
  const int n_pos = __ldg(n_dev);
  if (b0 >= n_pos) return;
  const int npos = n_pos - b0 < hp ? n_pos - b0 : hp;
  for (int i = tid; i < n_out * c_in; i += 256) { const int o = i / c_in, c = i % c_in; wsm[((c >> 3) * n_out + o) * 8 + (c & 7)] = __ldg(wh + i); }
  __syncthreads();
  for (int item = tid; item < npos * 90; item += 256) {
    const int p = item / 90, pix = item % 90;
    const size_t row = ((size_t)(b0 + p) * 90 + pix) * c_in;
    for (int o0 = 0; o0 < n_out; o0 += 6) {                  // six outputs per pass over the pixel's row (the row stays in L1)
      float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
      for (int g = 0; g < c_in / 8; ++g) {
        float x[8];
        if (act32) {
          const float4* a4 = reinterpret_cast<const float4*>(act32 + row + g * 8);
          const float4 u = __ldg(a4), w4 = __ldg(a4 + 1);
          x[0] = u.x; x[1] = u.y; x[2] = u.z; x[3] = u.w; x[4] = w4.x; x[5] = w4.y; x[6] = w4.z; x[7] = w4.w;
        } else {
          const uint4 v = __ldg(reinterpret_cast<const uint4*>(act + row + g * 8));
          const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
          for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); x[2 * j] = f.x; x[2 * j + 1] = f.y; }
        }
#pragma unroll
        for (int o = 0; o < 6; ++o) {
          if (o0 + o < n_out) {
            const float* wp = wsm + (g * n_out + o0 + o) * 8;
            const float4 wa = *reinterpret_cast<const float4*>(wp), wb = *reinterpret_cast<const float4*>(wp + 4);
            s[o] += x[0] * wa.x + x[1] * wa.y + x[2] * wa.z + x[3] * wa.w + x[4] * wb.x + x[5] * wb.y + x[6] * wb.z + x[7] * wb.w;
          }
        }
      }
#pragma unroll
      for (int o = 0; o < 6; ++o)
        if (o0 + o < n_out) feat[(p * n_out + o0 + o) * 90 + pix] = fmaxf(s[o] + __ldg(shifth + o0 + o), 0.f);
    }
  }
  __syncthreads();
  const int pol_in = pol_c * 90, pol_k = 3 * pol_k1;
  for (int i = tid; i < npos * pol_k1; i += 256) {
    const int p = i / pol_k1, k = i % pol_k1;
    const float f = k < pol_in ? feat[(p * n_out + k / 90) * 90 + k % 90] : 0.f;      // Keras Flatten of channels_first: c*90 + pix
    const __half hi = __float2half_rn(f);
    const __half lo = __float2half_rn(f - __half2float(hi));
    __half* row = pol_feat + (size_t)(b0 + p) * pol_k;
    row[k] = hi; row[pol_k1 + k] = lo; row[2 * pol_k1 + k] = hi;
  }
  float h[kHeadPos];
#pragma unroll
  for (int p = 0; p < kHeadPos; ++p) h[p] = 0.f;
  if (tid < hidden) {
    float acc[kHeadPos];
    const float bb = bv1[tid];
#pragma unroll
    for (int p = 0; p < kHeadPos; ++p) acc[p] = bb;
#pragma unroll 10
    for (int i = 0; i < val_c * 90; ++i) {
      const float wv = __ldg(wv1 + (size_t)i * hidden + tid);
#pragma unroll
      for (int p = 0; p < kHeadPos; ++p) acc[p] += feat[(p * n_out + pol_c + i / 90) * 90 + i % 90] * wv;
    }
    const float w2 = wv2[tid];
#pragma unroll
    for (int p = 0; p < kHeadPos; ++p) h[p] = fmaxf(acc[p], 0.f) * w2;
  }
#pragma unroll
  for (int p = 0; p < kHeadPos; ++p) {
    float v = h[p];
    for (int m = 16; m; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    if (lane == 0) red[p * 8 + warp] = v;
  }
  __syncthreads();
  if (tid < npos) {
    float sum = bv2[0];
    for (int i = 0; i < 8; ++i) sum += red[tid * 8 + i];
    value[b0 + tid] = tanhf(sum);
  }
}

// Softmax over the 2086 labels, finished from the per-N-tile statistics the policy GEMM epilogue wrote:
//   stats[row][t] = {m_t = max_j x_j, s_t = sum_j exp(x_j - m_t)} over the valid columns of tile t
//   m = max_t m_t,  S = sum_t s_t * exp(m_t - m),  p_j = exp(x_j - m) * (1 / S)
// `policy_prob` is the ONE definition of a policy probability in this library: k_softmax (the [B][2086] vector the
// reference-facing API returns) and k_legal_priors (only the legal moves of a search leaf) both evaluate it, so the
// integrated search sees bit for bit the numbers an external caller of cz_nn_forward would feed back.
struct RowStat { float mx, inv; };
__device__ __forceinline__ RowStat combine_stats(const float2* __restrict__ st, int n_tiles) {
  float mx = -INFINITY;
  for (int t = 0; t < n_tiles; ++t) mx = fmaxf(mx, __ldg(&st[t].x));
  float s = 0.f;
  for (int t = 0; t < n_tiles; ++t) { const float2 v = __ldg(st + t); s = __fmaf_rn(v.y, expf(v.x - mx), s); }
  RowStat r; r.mx = mx; r.inv = __frcp_rn(s);
  return r;
}
__device__ __forceinline__ float policy_prob(float logit, const RowStat& r) { return __fmul_rn(expf(logit - r.mx), r.inv); }

// logits [B][ldl] f32 -> policy [B][2086] f32. grid = batch, block = 256.
__global__ void __launch_bounds__(256) k_softmax(const float* __restrict__ logits, int ldl, const float2* __restrict__ stats, int n_tiles,
                                                  float* __restrict__ policy) {
  const int b = blockIdx.x;
  const RowStat rs = combine_stats(stats + (size_t)b * n_tiles, n_tiles);
  const float* l = logits + (size_t)b * ldl;
  for (int i = threadIdx.x; i < kLabels; i += 256) policy[(size_t)b * kLabels + i] = policy_prob(l[i], rs);
}

// Integrated search: softmax probabilities of the LEGAL moves of every leaf only (player.py:272-284 reads nothing else of the
// policy vector).  labels [n][CZ_MAX_MOVES] int16 (-1 = the move has no label), counts [n]; out [n][CZ_MAX_MOVES] f32.  Warp per leaf.
// kMirror (cz_config.eval_mirror): rows n..2n-1 are the leaves' mirrors; the prior is 0.5 * (p_leaf[lab] + p_{n+leaf}[M lab])
// and value[leaf] = 0.5 * (value2[leaf] + value2[n + leaf]), each sum and product rounded once.
template <bool kMirror>
__global__ void __launch_bounds__(128) k_legal_priors(const float* __restrict__ logits, int ldl, const float2* __restrict__ stats, int n_tiles,
                                                       const int16_t* __restrict__ labels, const int32_t* __restrict__ counts,
                                                       const int* __restrict__ n_dev, float* __restrict__ out,
                                                       const int16_t* __restrict__ mirror_lut, const float* __restrict__ value2,
                                                       float* __restrict__ value) {
  const int leaf = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n = __ldg(n_dev);
  if (leaf >= n) return;
  const RowStat rs = combine_stats(stats + (size_t)leaf * n_tiles, n_tiles);
  const float* l = logits + (size_t)leaf * ldl;
  RowStat rm{};
  const float* lm = nullptr;
  if (kMirror) {
    rm = combine_stats(stats + (size_t)(n + leaf) * n_tiles, n_tiles);
    lm = logits + (size_t)(n + leaf) * ldl;
    if (lane == 0) value[leaf] = __fmul_rn(0.5f, __fadd_rn(value2[leaf], value2[n + leaf]));
  }
  const int L = counts[leaf];
  for (int i = lane; i < L; i += 32) {
    const int lab = labels[(size_t)leaf * CZ_MAX_MOVES + i];
    float p = 0.f;
    if (lab >= 0) {
      p = policy_prob(l[lab], rs);
      if (kMirror) p = __fmul_rn(0.5f, __fadd_rn(p, policy_prob(lm[__ldg(mirror_lut + lab)], rm)));
    }
    out[(size_t)leaf * CZ_MAX_MOVES + i] = p;
  }
}
__global__ void k_set_int(int* p, int v) { *p = v; }

// Profiling bracket around the residual tower (nn_profile): one thread each, ordered by the stream.  Kernel nodes rather
// than event records, so that a WHILE node's body graph can hold them.  prof = {start, ns, brackets, positions}.
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__global__ void k_prof_begin(unsigned long long* prof) { prof[0] = global_ns(); }
__global__ void k_prof_end(unsigned long long* prof, const int* __restrict__ n_dev) {
  prof[1] += global_ns() - prof[0];
  prof[2] += 1;
  prof[3] += (unsigned long long)*n_dev;
}

// ---- weight preparation (Keras layout f32 -> folded operands)
__global__ void k_bn_fold(const float* gamma, const float* beta, const float* mean, const float* var, float* scale,
                          float* shift, int c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < c) {
    const float s = gamma[i] / sqrtf(var[i] + kBnEps);
    scale[i] = s;
    shift[i] = beta[i] - mean[i] * s;
  }
}
// HWIO [kh][kw][ci][co] -> same layout fp16 with scale[co] folded (first conv)
__global__ void k_prep_hwio(const float* w, const float* scale, __half* out, long long n, int co) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __float2half_rn(w[i] * scale[i % co]);
}
// HWIO [3][3][ci][co] -> [tap][co][ci] fp16, scale[co] folded (B operand, K-major)
__global__ void k_prep_conv3(const float* w, const float* scale, __half* out, int c) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = 9LL * c * c;
  if (i < n) {
    const int ci = (int)(i % c), co = (int)((i / c) % c), tap = (int)(i / ((long long)c * c));
    out[i] = __float2half_rn(w[((long long)tap * c + ci) * c + co] * scale[co]);
  }
}
// 1x1 conv HWIO [1][1][ci][co] -> [co][ci] f32 rows at out_row0.., scale folded
__global__ void k_prep_1x1(const float* w, const float* scale, float* out, int ci_n, int co_n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ci_n * co_n) {
    const int ci = i % ci_n, co = i / ci_n;
    out[(size_t)co * ci_n + ci] = w[(size_t)ci * co_n + co] * scale[co];
  }
}
// Dense (in,out) [pol_in][2086] -> [kPolN][3 * pol_k1] fp16 (zero padded), K-major, split as [w_hi | w_hi | w_lo]
__global__ void k_prep_policy(const float* w, __half* out, int pol_in, int pol_k1) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (long long)kPolN * pol_k1) {
    const int k = (int)(i % pol_k1), n = (int)(i / pol_k1);
    const float f = (k < pol_in && n < kLabels) ? w[(size_t)k * kLabels + n] : 0.f;
    const __half hi = __float2half_rn(f);
    const __half lo = __float2half_rn(f - __half2float(hi));
    __half* row = out + (size_t)n * 3 * pol_k1;
    row[k] = hi; row[pol_k1 + k] = hi; row[2 * pol_k1 + k] = lo;
  }
}
__global__ void k_copy_pad(const float* src, float* dst, int n_src, int n_dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_dst) dst[i] = i < n_src ? src[i] : 0.f;
}

// ------------------------------------------------------------------------------------------------
// One network's folded weights and their tensor maps (the arena holds two: best vs next generation,
// worker/evaluator.py:28-82).  nn_create fixes the buffers and maps for the runtime's lifetime: the search's captured graphs
// hold them by value, so cz_nn_set_weights may reload a network without a re-capture.
struct NetWeights {
  __half* w_first; float* shift_first;
  __half* w_conv;  float* shift_conv;      // [2*blocks][9*C*C], [2*blocks][C]
  float *wh, *shifth, *wv1, *bv1, *wv2, *bv2;
  __half* w_pol; float* b_pol;
  CUtensorMap map_wpol;
  std::vector<CUtensorMap> map_w;          // box rows = conv_tile_n(C, false)
  std::vector<CUtensorMap> map_w_64;       // box rows = 64: 64-column tiles of the small-batch launches (use_n_split)
  bool ready;                              // weights set (nn_set_weights)
};

struct NnRuntime {
  int filters, blocks, value_fc, max_batch;
  int pol_c, val_c, pol_k1;               // head widths (policy / value conv channels) and the padded policy feature count
  NetWeights nets[2]; int n_nets;
  cudaStream_t stream;
  uint64_t launches;
  // activations
  __half *x, *t, *y, *pol_feat;
  float *x32, *y32;                      // fp32 skip stream
  float* logits;
  float2* stats;                         // [max_batch][kPolN / 256] softmax statistics of the policy GEMM's N tiles
  int* n_scalar;                         // device copy of a host-known batch size (reference-facing forward)
  bool heads_attr;                       // k_heads was granted > 48 KB of dynamic shared memory (wide legacy heads)
  uint8_t* boards_tmp;
  int in_planes;                         // 14, or 28 with use_history (board + history board per position)
  float* scratch;                            // 2*C floats for BN folding
  CUtensorMap map_pf;                    // policy GEMM operand (pol_feat)
  bool fp32_skip;                        // keep the residual (skip) stream in fp32: halves the value error of deep nets, ~+30 % time
  CUtensorMap hmap_x, hmap_t, hmap_y;    // the three activation buffers as the conv's halo loads read them
  CUtensorMap emap_t;                    // conv1's output buffer as the staged conv epilogue stores it
  // optional timing of the residual tower (bench.py roofline): with `profile` on, every forward brackets its tower with
  // k_prof_begin / k_prof_end, which accumulate into prof[4] = {start, ns, brackets, positions}
  bool profile;
  unsigned long long* prof;
};

static void layout(NnRuntime* r, Carver& cv) {
  const int c = r->filters;
  const size_t act = (size_t)r->max_batch * 90 * c;       // elements of one activation buffer
  r->x = (__half*)cv.take(act * sizeof(__half));
  r->t = (__half*)cv.take(act * sizeof(__half));
  r->y = (__half*)cv.take(act * sizeof(__half));
  r->x32 = (float*)cv.take(act * sizeof(float));
  r->y32 = (float*)cv.take(act * sizeof(float));
  r->pol_feat = (__half*)cv.take(((size_t)r->max_batch + 128) * 3 * r->pol_k1 * sizeof(__half));
  r->logits = (float*)cv.take((size_t)r->max_batch * kPolN * sizeof(float));
  r->stats = (float2*)cv.take((size_t)r->max_batch * (kPolN / 256) * sizeof(float2));
  r->n_scalar = (int*)cv.take(64);
  r->boards_tmp = (uint8_t*)cv.take((size_t)r->max_batch * 2 * CZ_BOARD_STRIDE);
  r->prof = (unsigned long long*)cv.take(4 * sizeof(unsigned long long));
  for (int k = 0; k < r->n_nets; ++k) {
    NetWeights& w = r->nets[k];
    w.w_first = (__half*)cv.take((size_t)25 * 28 * c * sizeof(__half));
    w.shift_first = (float*)cv.take(c * sizeof(float));
    w.w_conv = (__half*)cv.take((size_t)2 * r->blocks * 9 * c * c * sizeof(__half));
    w.shift_conv = (float*)cv.take((size_t)2 * r->blocks * c * sizeof(float));
    w.wh = (float*)cv.take((size_t)(r->pol_c + r->val_c) * c * sizeof(float));
    w.shifth = (float*)cv.take((size_t)(r->pol_c + r->val_c + 4) * sizeof(float));
    w.wv1 = (float*)cv.take((size_t)r->val_c * 90 * r->value_fc * sizeof(float));
    w.bv1 = (float*)cv.take(r->value_fc * sizeof(float));
    w.wv2 = (float*)cv.take(r->value_fc * sizeof(float));
    w.bv2 = (float*)cv.take(4 * sizeof(float));
    w.w_pol = (__half*)cv.take((size_t)kPolN * 3 * r->pol_k1 * sizeof(__half));
    w.b_pol = (float*)cv.take(kPolN * sizeof(float));
  }
  r->scratch = (float*)cv.take((size_t)(2 * 256 + 2 * kMaxHeadOut) * sizeof(float));
}

static void set_heads(NnRuntime* r, int pol_c, int val_c) {
  r->pol_c = pol_c > 0 ? pol_c : 4; r->val_c = val_c > 0 ? val_c : 2;     // agent/model.py:47-61 defaults
  r->pol_k1 = (r->pol_c * 90 + 63) / 64 * 64;
}
size_t nn_workspace_bytes(int filters, int blocks, int value_fc, int max_batch, int n_nets, int pol_c, int val_c) {
  NnRuntime tmp;
  tmp.filters = filters; tmp.blocks = blocks; tmp.value_fc = value_fc; tmp.max_batch = max_batch; tmp.n_nets = n_nets;
  set_heads(&tmp, pol_c, val_c);
  Carver cv{nullptr, 0};
  layout(&tmp, cv);
  return cv.off + 4096;
}

NnRuntime* nn_create(int device, int filters, int blocks, int value_fc, int max_batch, void* workspace, size_t bytes,
                     void* stream, int fp32_skip_mode, int n_nets, int in_planes, int pol_c, int val_c) {
  (void)device;
  if (filters % 64 != 0 || filters < 64 || filters > 256) { cz_fail(CZ_ERR_UNSUPPORTED, "nn: filters must be 64..256 step 64"); return nullptr; }
  if (value_fc > 256 || value_fc < 1) { cz_fail(CZ_ERR_UNSUPPORTED, "nn: value_fc_size must be <= 256"); return nullptr; }
  if (n_nets < 1 || n_nets > 2) { cz_fail(CZ_ERR_ARG, "nn: 1 or 2 networks"); return nullptr; }
  if (pol_c < 0 || val_c < 0 || pol_c > 32 || val_c > 4 || (pol_c > 0 ? pol_c : 4) + (val_c > 0 ? val_c : 2) > kMaxHeadOut) {
    cz_fail(CZ_ERR_UNSUPPORTED, "nn: head widths up to 32 policy / 4 value channels"); return nullptr;
  }
  if (bytes < nn_workspace_bytes(filters, blocks, value_fc, max_batch, n_nets, pol_c, val_c)) { cz_fail(CZ_ERR_ARG, "nn: workspace too small"); return nullptr; }
  NnRuntime* r = new NnRuntime();
  set_heads(r, pol_c, val_c);
  r->heads_attr = false;
  r->filters = filters; r->blocks = blocks; r->value_fc = value_fc; r->max_batch = max_batch; r->n_nets = n_nets;
  r->stream = (cudaStream_t)stream; r->launches = 0;
  r->in_planes = in_planes == 28 ? 28 : 14;
  // 0 = auto (fp32 skip stream for towers of 10 blocks and more, where fp16 rounding of the skip stream pushes the outputs
  // past 1e-3: value 1.1e-3 .. 1.5e-3 at 20 random-init blocks vs <= 6e-4 with fp32; policy 1.6e-3 vs 9.8e-4 on the
  // reference's trained 192x10 net), 1 = always, 2 = never
  r->fp32_skip = fp32_skip_mode == 1 || (fp32_skip_mode == 0 && blocks >= 10);
  r->profile = false;
  Carver cv{(uint8_t*)workspace, 0};
  layout(r, cv);
  const int c = filters;
  int rc = 0;
  rc |= make_map_2d(&r->hmap_x, r->x, c, (long long)max_batch * 90, igemm::kHaloBox);
  rc |= make_map_2d(&r->hmap_t, r->t, c, (long long)max_batch * 90, igemm::kHaloBox);
  rc |= make_map_2d(&r->hmap_y, r->y, c, (long long)max_batch * 90, igemm::kHaloBox);
  rc |= make_map_epi(&r->emap_t, r->t, c, (long long)max_batch * 90);
  rc |= make_map_2d(&r->map_pf, r->pol_feat, 3 * r->pol_k1, (long long)max_batch + 128, 128);
  for (int k = 0; k < n_nets; ++k) {
    NetWeights& w = r->nets[k];
    w.ready = false;
    rc |= make_map_2d(&w.map_wpol, w.w_pol, 3 * r->pol_k1, kPolN, 256);
    w.map_w.resize(2 * blocks);
    w.map_w_64.resize(2 * blocks);
    for (int i = 0; i < 2 * blocks; ++i) {
      rc |= make_map_2d(&w.map_w[i], w.w_conv + (size_t)i * 9 * c * c, c, 9LL * c, conv_tile_n(c, false));
      rc |= make_map_2d(&w.map_w_64[i], w.w_conv + (size_t)i * 9 * c * c, c, 9LL * c, 64);
    }
  }
  if (rc) { delete r; return nullptr; }
  // the last, partial M tile of a conv or of the policy GEMM loads rows past the batch: they start as zeros, not as whatever
  // the workspace held
  cudaMemsetAsync(r->x, 0, (size_t)max_batch * 90 * c * 2, r->stream);
  cudaMemsetAsync(r->t, 0, (size_t)max_batch * 90 * c * 2, r->stream);
  cudaMemsetAsync(r->y, 0, (size_t)max_batch * 90 * c * 2, r->stream);
  cudaMemsetAsync(r->pol_feat, 0, ((size_t)max_batch + 128) * 3 * r->pol_k1 * 2, r->stream);
  cudaMemsetAsync(r->prof, 0, 4 * sizeof(unsigned long long), r->stream);
  return r;
}

void nn_destroy(NnRuntime* r) { delete r; }
void nn_profile(NnRuntime* r, bool on) { if (r) { r->profile = on; } }
// Synchronises the stream.  ms = device time spent in the residual towers bracketed since the last read, launches = their
// igemm launches, flops = their algorithmic flops (2*90*9*C*C per position per conv); clears the accumulators.
int nn_profile_read(NnRuntime* r, double* ms, uint64_t* launches, double* flops) {
  if (!r) return cz_fail(CZ_ERR_STATE, "no network");
  unsigned long long p[4];
  CZ_CUDA(cudaMemcpyAsync(p, r->prof, sizeof(p), cudaMemcpyDeviceToHost, r->stream));
  CZ_CUDA(cudaMemsetAsync(r->prof, 0, sizeof(p), r->stream));
  CZ_CUDA(cudaStreamSynchronize(r->stream));
  if (ms) *ms = (double)p[1] * 1e-6;
  if (launches) *launches = p[2] * (uint64_t)(2 * r->blocks);
  if (flops) *flops = (double)p[3] * (2.0 * 90.0 * 9.0 * r->filters * r->filters * 2.0 * r->blocks);
  return 0;
}
bool nn_ready(const NnRuntime* r) {
  if (!r) return false;
  for (int k = 0; k < r->n_nets; ++k)
    if (!r->nets[k].ready) return false;
  return true;
}
// Network `net` of r if its weights are set; null (and cz_last_error says why) otherwise.
static const NetWeights* ready_net(NnRuntime* r, int net) {
  if (!r || net < 0 || net >= r->n_nets) { cz_fail(CZ_ERR_STATE, "no such network"); return nullptr; }
  if (!r->nets[net].ready) { cz_fail(CZ_ERR_STATE, "network weights not set (cz_nn_set_weights)"); return nullptr; }
  return &r->nets[net];
}
uint64_t nn_launches(const NnRuntime* r) { return r ? r->launches : 0; }

// ---- weights -----------------------------------------------------------------------------------
const cz_tensor_desc* find_keras_tensor(const cz_tensor_desc* descs, int n, const std::string& layer, const std::string& weight) {
  for (int i = 0; i < n; ++i) {
    std::string nm = descs[i].name ? descs[i].name : "";
    const size_t slash = nm.find('/');
    if (slash == std::string::npos) continue;
    std::string l = nm.substr(0, slash), w = nm.substr(slash + 1);
    const size_t colon = w.find(':');
    if (colon != std::string::npos) w = w.substr(0, colon);
    const size_t s2 = w.find('/');            // "layer/layer/kernel" style
    if (s2 != std::string::npos) w = w.substr(s2 + 1);
    if (w != weight) continue;
    if (l == layer || (l.size() > layer.size() && l.compare(0, layer.size(), layer) == 0 && l[layer.size()] == '-')) return &descs[i];
  }
  return nullptr;
}

#define NEED(var, layer, weight, count)                                                                      \
  const cz_tensor_desc* var = find_keras_tensor(descs, n_descs, layer, weight);                              \
  if (!var || var->numel != (long long)(count))                                                              \
    return cz_fail(CZ_ERR_ARG, "cz_nn_set_weights: missing or mis-sized tensor %s/%s (want %lld)", std::string(layer).c_str(), weight, (long long)(count));

static int fold_bn(NnRuntime* r, const cz_tensor_desc* descs, int n_descs, const std::string& layer, int c, float* scale, float* shift) {
  NEED(g, layer, "gamma", c);
  NEED(b, layer, "beta", c);
  NEED(m, layer, "moving_mean", c);
  NEED(v, layer, "moving_variance", c);
  k_bn_fold<<<(c + 127) / 128, 128, 0, r->stream>>>((const float*)g->dev, (const float*)b->dev, (const float*)m->dev,
                                                     (const float*)v->dev, scale, shift, c);
  r->launches++;
  return 0;
}

int nn_set_weights(NnRuntime* r, int net, const cz_tensor_desc* descs, int n_descs) {
  if (!r) return cz_fail(CZ_ERR_STATE, "cz_nn_set_weights: engine was created without a network (nn_filters = 0)");
  if (net < 0 || net >= r->n_nets) return cz_fail(CZ_ERR_ARG, "cz_nn_set_weights: network %d of %d", net, r->n_nets);
  NetWeights& w = r->nets[net];
  const int c = r->filters;
  cudaStream_t st = r->stream;
  float* scale = r->scratch;
  {
    NEED(k, "input_conv", "kernel", 25LL * r->in_planes * c);
    if (fold_bn(r, descs, n_descs, "input_batchnorm", c, scale, w.shift_first)) return CZ_ERR_ARG;
    const long long nn = 25LL * r->in_planes * c;
    k_prep_hwio<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>((const float*)k->dev, scale, w.w_first, nn, c);
  }
  for (int i = 0; i < r->blocks; ++i) {
    for (int j = 0; j < 2; ++j) {
      const std::string conv = "res" + std::to_string(i + 1) + "_conv" + std::to_string(j + 1);
      const std::string bn = "res" + std::to_string(i + 1) + "_batchnorm" + std::to_string(j + 1);
      NEED(k, conv, "kernel", 9LL * c * c);
      const int li = 2 * i + j;
      if (fold_bn(r, descs, n_descs, bn, c, scale, w.shift_conv + (size_t)li * c)) return CZ_ERR_ARG;
      const long long nn = 9LL * c * c;
      k_prep_conv3<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>((const float*)k->dev, scale, w.w_conv + (size_t)li * nn, c);
    }
  }
  {
    const int pc = r->pol_c, vc = r->val_c;
    NEED(kp, "policy_conv", "kernel", (long long)pc * c);
    if (fold_bn(r, descs, n_descs, "policy_batchnorm", pc, scale, w.shifth)) return CZ_ERR_ARG;
    k_prep_1x1<<<(pc * c + 255) / 256, 256, 0, st>>>((const float*)kp->dev, scale, w.wh, c, pc);
    NEED(kv, "value_conv", "kernel", (long long)vc * c);
    float* scale_v = r->scratch + 2 * 256 + kMaxHeadOut;     // k_bn_fold of the policy head above may still be reading `scale`
    if (fold_bn(r, descs, n_descs, "value_batchnorm", vc, scale_v, w.shifth + pc)) return CZ_ERR_ARG;
    k_prep_1x1<<<(vc * c + 255) / 256, 256, 0, st>>>((const float*)kv->dev, scale_v, w.wh + (size_t)pc * c, c, vc);
  }
  {
    NEED(k, "policy_out", "kernel", (long long)r->pol_c * 90 * kLabels);
    NEED(b, "policy_out", "bias", kLabels);
    const long long nn = (long long)kPolN * r->pol_k1;
    k_prep_policy<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>((const float*)k->dev, w.w_pol, r->pol_c * 90, r->pol_k1);
    k_copy_pad<<<(kPolN + 255) / 256, 256, 0, st>>>((const float*)b->dev, w.b_pol, kLabels, kPolN);
  }
  {
    const int h = r->value_fc;
    NEED(k1, "value_dense", "kernel", (long long)r->val_c * 90 * h);
    NEED(b1, "value_dense", "bias", h);
    NEED(k2, "value_out", "kernel", h);
    NEED(b2, "value_out", "bias", 1);
    CZ_CUDA(cudaMemcpyAsync(w.wv1, k1->dev, (size_t)r->val_c * 90 * h * 4, cudaMemcpyDeviceToDevice, st));
    CZ_CUDA(cudaMemcpyAsync(w.bv1, b1->dev, (size_t)h * 4, cudaMemcpyDeviceToDevice, st));
    CZ_CUDA(cudaMemcpyAsync(w.wv2, k2->dev, (size_t)h * 4, cudaMemcpyDeviceToDevice, st));
    CZ_CUDA(cudaMemcpyAsync(w.bv2, b2->dev, 4, cudaMemcpyDeviceToDevice, st));
  }
  r->launches += 6 + 2 * r->blocks;
  CZ_CUDA(cudaGetLastError());
  CZ_CUDA(cudaStreamSynchronize(st));
  w.ready = true;
  return 0;
}

// ---- forward -----------------------------------------------------------------------------------
// One pass over at most `n_max` positions; the ACTUAL batch size is the device integer *n_dev (every launch has a fixed
// shape sized for n_max, kernels read *n_dev and leave the rest untouched), so a search never has to tell the host how
// many leaves a wave produced.  Leaves logits [n][kPolN] + per-tile softmax statistics in r->logits / r->stats.
static int conv_first_threads(int c) {                    // (c/2) channel pairs x as many pixel groups as fit 256 threads
  const int pairs = c / 2;
  int g = 256 / pairs;
  if (g < 1) g = 1;
  while (pairs * g < 96) ++g;                             // phase 1 needs 90 threads
  return pairs * g;
}
static int fw_first(NnRuntime* r, const NetWeights& w, const uint8_t* boards, int n, const int* n_dev) {
  const int c = r->filters;
  const bool s32 = r->fp32_skip;
  int slices = (2 * num_sms() + n - 1) / n;                // >= 2 CTAs per SM in flight; big batches: one CTA per position
  if (slices > 15) slices = 15;
  k_conv_first<<<dim3(n, slices), conv_first_threads(c), 0, r->stream>>>(boards, w.w_first, w.shift_first, r->x, s32 ? r->x32 : nullptr, c,
                                                            r->in_planes, (r->in_planes / 14) * CZ_BOARD_STRIDE, n_dev);
  r->launches++;
  CZ_CUDA(cudaGetLastError());
  return 0;
}
static int fw_tower(NnRuntime* r, const NetWeights& w, int n, const int* n_dev) {
  const int c = r->filters;
  cudaStream_t st = r->stream;
  float *x32 = r->fp32_skip ? r->x32 : nullptr, *y32 = r->fp32_skip ? r->y32 : nullptr;
  CUtensorMap *ix = &r->hmap_x, *iy = &r->hmap_y;
  __half *x = r->x, *y = r->y;
  const bool split = use_n_split(n, c);
  const int nt = conv_tile_n(c, split);
  const std::vector<CUtensorMap>& wm = split ? w.map_w_64 : w.map_w;
  for (int i = 0; i < r->blocks; ++i) {
    // conv1: x -> t (no skip);  conv2: t (+ skip x or x32) -> y (+ y32)
    igemm::Args d1 = conv_args(n, c, w.shift_conv + (size_t)(2 * i) * c, nullptr, r->t, 1, split);
    igemm::Args d2 = conv_args(n, c, w.shift_conv + (size_t)(2 * i + 1) * c, x, y, 1, split);
    d1.n_dev = d2.n_dev = n_dev;
    d2.residual32 = x32; d2.out32 = y32;
    if (launch_igemm(nt, *ix, wm[2 * i], d1, st, &r->emap_t)) return CZ_ERR_CUDA;
    if (launch_igemm(nt, r->hmap_t, wm[2 * i + 1], d2, st)) return CZ_ERR_CUDA;
    r->launches += 2;
    std::swap(x, y); std::swap(x32, y32); std::swap(ix, iy);
  }
  return 0;
}
static int fw_heads(NnRuntime* r, const NetWeights& w, int n, const int* n_dev, float* value) {
  const int c = r->filters;
  const bool s32 = r->fp32_skip;
  const bool odd = (r->blocks & 1) != 0;                   // the tower ping-pongs x <-> y once per block
  const __half* x = odd ? r->y : r->x;
  const float* x32 = s32 ? (odd ? r->y32 : r->x32) : nullptr;
  const size_t hsm = heads_smem_bytes(c, r->pol_c + r->val_c);
  if (hsm > 48 * 1024 && !r->heads_attr) {
    CZ_CUDA(cudaFuncSetAttribute(k_heads, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hsm));
    r->heads_attr = true;
  }
  const int hp = n <= 2 * num_sms() ? 1 : kHeadPos;       // small batches: a block per position (same arithmetic per position)
  k_heads<<<(n + hp - 1) / hp, 256, hsm, r->stream>>>(x, x32, c, n_dev, r->pol_c, r->val_c, r->pol_k1, w.wh, w.shifth,
                                                      w.wv1, w.bv1, w.wv2, w.bv2, r->value_fc, r->pol_feat, value, hp);
  igemm::Args ap = dense_args(n, kLabels, kPolN, 3 * r->pol_k1, 256, w.b_pol, r->logits, kPolN);
  ap.n_dev = n_dev; ap.rows_per_unit = 1; ap.row_stats = r->stats;
  if (launch_igemm(256, r->map_pf, w.map_wpol, ap, r->stream)) return CZ_ERR_CUDA;
  r->launches += 2;
  CZ_CUDA(cudaGetLastError());
  return 0;
}
// first conv, residual tower (bracketed by k_prof_begin / k_prof_end while profiling is on), heads + policy GEMM
static int forward_tower(NnRuntime* r, const NetWeights& w, const uint8_t* boards, int n_max, const int* n_dev, float* value) {
  int rc = fw_first(r, w, boards, n_max, n_dev);
  if (rc) return rc;
  if (r->profile) k_prof_begin<<<1, 1, 0, r->stream>>>(r->prof);
  rc = fw_tower(r, w, n_max, n_dev);
  if (rc) return rc;
  if (r->profile) {
    k_prof_end<<<1, 1, 0, r->stream>>>(r->prof, n_dev);
    r->launches += 2;
  }
  return fw_heads(r, w, n_max, n_dev, value);
}

// host-known batch: the reference-facing predict_on_batch (api.py:62-64) -> the full softmax vector
static int forward_chunk(NnRuntime* r, const NetWeights& w, const uint8_t* boards, int n, float* policy, float* value) {
  k_set_int<<<1, 1, 0, r->stream>>>(r->n_scalar, n);
  const int rc = forward_tower(r, w, boards, n, r->n_scalar, value);
  if (rc) return rc;
  k_softmax<<<n, 256, 0, r->stream>>>(r->logits, kPolN, r->stats, kPolN / 256, policy);
  r->launches += 2;
  CZ_CUDA(cudaGetLastError());
  return 0;
}

int nn_forward_boards(NnRuntime* r, int net, const uint8_t* boards, int batch, float* policy, float* value) {
  const NetWeights* w = ready_net(r, net);
  if (!w) return CZ_ERR_STATE;
  for (int off = 0; off < batch; off += r->max_batch) {
    const int n = batch - off < r->max_batch ? batch - off : r->max_batch;
    const int rc = forward_chunk(r, *w, boards + (size_t)off * (r->in_planes / 14) * CZ_BOARD_STRIDE, n, policy + (size_t)off * kLabels, value + off);
    if (rc) return rc;
  }
  return 0;
}

int nn_forward_planes(NnRuntime* r, int net, const float* planes, int batch, float* policy, float* value) {
  const NetWeights* w = ready_net(r, net);
  if (!w) return CZ_ERR_STATE;
  for (int off = 0; off < batch; off += r->max_batch) {
    const int n = batch - off < r->max_batch ? batch - off : r->max_batch;
    k_planes_to_boards<<<n, 96, 0, r->stream>>>(planes + (size_t)off * r->in_planes * 90, r->boards_tmp, n, r->in_planes);
    r->launches++;
    const int rc = forward_chunk(r, *w, r->boards_tmp, n, policy + (size_t)off * kLabels, value + off);
    if (rc) return rc;
  }
  return 0;
}

// The search's evaluation step: up to n_max leaves (actual count *n_dev), boards + legal-move labels in, value [n] and the
// softmax probabilities of the legal moves [n][CZ_MAX_MOVES] out.  Fixed launch shapes: safe to capture into a CUDA graph.
int nn_forward_leaves(NnRuntime* r, int net, const uint8_t* boards, int n_max, const int* n_dev, const int16_t* labels,
                      const int32_t* label_counts, float* legal_p, float* value, const int16_t* mirror_lut, float* value2) {
  const NetWeights* w = ready_net(r, net);
  if (!w) return CZ_ERR_STATE;
  const bool mirror = mirror_lut != nullptr;
  const int rows = mirror ? 2 * n_max : n_max;
  if (rows > r->max_batch) return cz_fail(CZ_ERR_ARG, "nn_forward_leaves: %d rows > max batch %d", rows, r->max_batch);
  if (mirror && !value2) return cz_fail(CZ_ERR_ARG, "nn_forward_leaves: the mirror form needs its value scratch");
  const int rc = forward_tower(r, *w, boards, rows, mirror ? n_dev + 2 : n_dev, mirror ? value2 : value);
  if (rc) return rc;
  if (mirror)
    k_legal_priors<true><<<(n_max + 3) / 4, 128, 0, r->stream>>>(r->logits, kPolN, r->stats, kPolN / 256, labels, label_counts, n_dev,
                                                                 legal_p, mirror_lut, value2, value);
  else
    k_legal_priors<false><<<(n_max + 3) / 4, 128, 0, r->stream>>>(r->logits, kPolN, r->stats, kPolN / 256, labels, label_counts, n_dev,
                                                                  legal_p, nullptr, nullptr, nullptr);
  r->launches++;
  CZ_CUDA(cudaGetLastError());
  return 0;
}
bool nn_profiling(const NnRuntime* r) { return r && r->profile; }
// Parity tests: copy rows of an intermediate buffer out after a forward.  Which physical buffer holds a stage follows the
// ping-pong of fw_tower and the choice fw_heads makes (x <-> y once per block, the fp32 copies alongside).  Off the forward
// path: nothing here runs unless a test asks.
int nn_read_buffer(NnRuntime* r, int which, int n, void* dst, long long dst_bytes, long long* row_bytes) {
  if (!r) return cz_fail(CZ_ERR_STATE, "cz_nn_read_buffer: engine has no network");
  const bool s32 = r->fp32_skip, odd = (r->blocks & 1) != 0;
  const long long act = 90LL * r->filters;
  const void* src = nullptr;
  long long row = 0;
  switch (which) {
    case CZ_NN_BUF_FIRST_OUT:
    case CZ_NN_BUF_FIRST_OUT32:
      if (r->blocks != 1) return cz_fail(CZ_ERR_STATE, "cz_nn_read_buffer: the first convolution's output survives only a 1-block tower");
      if (which == CZ_NN_BUF_FIRST_OUT32 && !s32) return cz_fail(CZ_ERR_STATE, "cz_nn_read_buffer: no fp32 skip stream");
      src = which == CZ_NN_BUF_FIRST_OUT ? (const void*)r->x : (const void*)r->x32;
      row = which == CZ_NN_BUF_FIRST_OUT ? act * 2 : act * 4;
      break;
    case CZ_NN_BUF_LAST_CONV1:
      if (r->blocks < 1) return cz_fail(CZ_ERR_STATE, "cz_nn_read_buffer: no residual block");
      src = r->t; row = act * 2;
      break;
    case CZ_NN_BUF_TOWER_OUT:
      src = odd ? r->y : r->x; row = act * 2;
      break;
    case CZ_NN_BUF_TOWER_OUT32:
      if (!s32) return cz_fail(CZ_ERR_STATE, "cz_nn_read_buffer: no fp32 skip stream");
      src = odd ? r->y32 : r->x32; row = act * 4;
      break;
    case CZ_NN_BUF_POL_FEAT: src = r->pol_feat; row = 3LL * r->pol_k1 * 2; break;
    case CZ_NN_BUF_LOGITS: src = r->logits; row = (long long)kPolN * 4; break;
    case CZ_NN_BUF_STATS: src = r->stats; row = (long long)(kPolN / 256) * 8; break;
    default: return cz_fail(CZ_ERR_ARG, "cz_nn_read_buffer: unknown buffer %d", which);
  }
  if (row_bytes) *row_bytes = row;
  if (!dst) return 0;
  if (n < 0 || n > r->max_batch) return cz_fail(CZ_ERR_ARG, "cz_nn_read_buffer: %d rows of a batch of at most %d", n, r->max_batch);
  if (dst_bytes < (long long)n * row) return cz_fail(CZ_ERR_ARG, "cz_nn_read_buffer: %lld bytes < %d rows x %lld", dst_bytes, n, row);
  CZ_CUDA(cudaMemcpyAsync(dst, src, (size_t)n * row, cudaMemcpyDeviceToDevice, r->stream));
  CZ_CUDA(cudaStreamSynchronize(r->stream));
  return 0;
}
int nn_launches_per_forward(const NnRuntime* r) { return r ? 1 + 2 * r->blocks + 3 + (r->profile ? 2 : 0) : 0; }

}  // namespace cznn

// ------------------------------------------------------------------------------------------------
// Building blocks exported for parity tests and profiling (not part of the reference-facing surface).
extern "C" {

// 3x3 "same" convolution on activations fp16 [n_boards][10][9][c], the tower's full-width conv tiles:
// out = relu?(conv(in, w) + bias (+ residual)); residual and out have the layout of in; w: fp16 [9][c_out = c][c_in = c],
// bias f32 [c].
int cz_igemm_conv3x3_dense(const void* act_in, const void* w, const float* bias, const void* residual, void* act_out,
                           int n_boards, int c, int relu, void* stream) {
  using namespace cznn;
  if (c % 64 || c < 64 || c > 256 || n_boards <= 0) return cz_fail(CZ_ERR_ARG, "cz_igemm_conv3x3_dense: bad shape");
  CUtensorMap ma, mb;
  if (make_map_2d(&ma, act_in, c, (long long)n_boards * 90, igemm::kHaloBox)) return CZ_ERR_CUDA;
  if (make_map_2d(&mb, w, c, 9LL * c, conv_tile_n(c, false))) return CZ_ERR_CUDA;
  igemm::Args a = conv_args(n_boards, c, bias, (const __half*)residual, act_out, relu);
  return launch_igemm(conv_tile_n(c, false), ma, mb, a, (cudaStream_t)stream);
}

// out[m][n] = sum_k a[m][k] * w[n][k] + bias[n]; a fp16 [m_alloc >= ceil128(m)][k], w fp16 [n_pad][k], k % 64 == 0,
// n_pad % n_tile == 0, out f32 [m][ldo].
int cz_igemm_dense(const void* a_dev, const void* w_dev, const float* bias, float* out, int m, int n_valid, int n_pad,
                   int k, int n_tile, int ldo, void* stream) {
  using namespace cznn;
  if (k % 64 || n_pad % n_tile || m <= 0) return cz_fail(CZ_ERR_ARG, "cz_igemm_dense: bad shape");
  CUtensorMap ma, mb;
  if (make_map_2d(&ma, a_dev, k, (long long)m, 128)) return CZ_ERR_CUDA;
  if (make_map_2d(&mb, w_dev, k, n_pad, n_tile)) return CZ_ERR_CUDA;
  igemm::Args a = dense_args(m, n_valid, n_pad, k, n_tile, bias, out, ldo);
  return launch_igemm(n_tile, ma, mb, a, (cudaStream_t)stream);
}

}  // extern "C"
