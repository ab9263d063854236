// cz_train.cu — one training step of the policy-value network (agent/model.py:32-83) on H100 (sm_90a): what Keras
// Model.fit runs per batch for worker/optimize.py:108-136.
//
//   forward (training mode)   planes -> one-hot gather 5x5 conv (raw) -> BN(batch stats) + ReLU
//                              per block: k_igemm 3x3 conv (raw fp32 out) -> BN + ReLU -> k_igemm -> BN + skip + ReLU
//                              heads: 1x1 convs, BN, ReLU, policy Dense + softmax + clipped CE, value MLP + tanh + MSE
//   backward                   heads (plain CUDA), per block: BN backward, wgrad (wgrad::k_wgrad), dgrad (k_igemm on
//                              tap-flipped weights), first-conv wgrad (gather-sum over the one-hot planes)
//   update                     L2 gradient 2*l2*K, SGD momentum on fp32 master weights, BN moving statistics
//
// Every reduction runs in a fixed order (per-CTA partials, then one ordered sum; no float atomics), so a step is
// bit-reproducible.  Gradient operands of the tensor-core convolutions are fp16 scaled by a power of two chosen from the
// tensor's own max|.|, and unscaled in fp32.  DESIGN.md §11 lists the Keras semantics restated here.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <string>
#include <vector>

#include "cz_err.h"
#include "cz_igemm.cuh"
#include "cz_nn.cuh"
#include "cz_nn_host.cuh"
#include "cz_wgrad.cuh"

namespace cztrain {

using cznn::Carver;

#define CZ_TRY(x)              \
  do {                         \
    const int r__ = (x);       \
    if (r__) return r__;       \
  } while (0)

constexpr int kLabels = CZ_N_LABELS;
constexpr float kBnEps = 1e-3f;
constexpr int kMaxSplits = 14;        // wgrad K splits
constexpr int kGemmMaxSplits = 64;
constexpr int kGemmPartFloats = kGemmMaxSplits * 70000;

static unsigned blocks_for(long long n, int threads = 256) {
  long long b = (n + threads - 1) / threads;
  return (unsigned)(b < 1 ? 1 : (b > 65535LL * 8 ? 65535LL * 8 : b));
}

// ------------------------------------------------------------------------------------------------ small kernels
// one-hot planes [B][in_planes][10][9] -> plane index per (position, board, pixel) (-1 = empty square)
__global__ void k_plane_index(const float* __restrict__ planes, int8_t* __restrict__ pl, int n, int in_planes) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nb = in_planes / 14;
  if (i >= (long long)n * nb * 90) return;
  const int pix = (int)(i % 90), h = (int)((i / 90) % nb);
  const long long b = i / (90 * nb);
  int8_t p = -1;
  for (int q = 0; q < 14; ++q)
    if (planes[(b * in_planes + h * 14 + q) * 90 + pix] > 0.5f) p = (int8_t)q;
  pl[(b * 2 + h) * 90 + pix] = p;
}

// 5x5 "same" input convolution without BN folding: z[b][pix][co] = sum over the occupied taps of w[tap][plane][co].
// grid = n, block = C threads (one output channel each).
__global__ void k_first_fwd(const int8_t* __restrict__ pl, const float* __restrict__ w, float* __restrict__ z, int c, int in_planes) {
  const int b = blockIdx.x, co = threadIdx.x, nb = in_planes / 14;
  __shared__ int8_t sp[2][90];
  for (int i = threadIdx.x; i < nb * 90; i += blockDim.x) sp[i / 90][i % 90] = pl[((size_t)b * 2 + i / 90) * 90 + i % 90];
  __syncthreads();
  if (co >= c) return;
  for (int pix = 0; pix < 90; ++pix) {
    const int r = pix / 9, col = pix % 9;
    float acc = 0.f;
    for (int kh = 0; kh < 5; ++kh) {
      const int rr = r + kh - 2;
      if (rr < 0 || rr > 9) continue;
      for (int kw = 0; kw < 5; ++kw) {
        const int cc = col + kw - 2;
        if (cc < 0 || cc > 8) continue;
        for (int h = 0; h < nb; ++h) {
          const int p = sp[h][rr * 9 + cc];
          if (p >= 0) acc += __ldg(w + ((size_t)(kh * 5 + kw) * in_planes + h * 14 + p) * c + co);
        }
      }
    }
    z[((size_t)b * 90 + pix) * c + co] = acc;
  }
}

// first-conv weight gradient: part[chunk][tap][plane][co] = sum over the chunk's positions and pixels whose tapped square
// holds `plane` of dz[b][pix][co].  grid = (25 taps, chunks), block = C threads; each thread owns its column of `acc`.
__global__ void k_first_wgrad(const int8_t* __restrict__ pl, const float* __restrict__ dz, float* __restrict__ part, int n,
                              int per_chunk, int c, int in_planes) {
  extern __shared__ float facc[];                      // [in_planes][C]
  const int tap = blockIdx.x, chunk = blockIdx.y, co = threadIdx.x, nb = in_planes / 14;
  const int kh = tap / 5, kw = tap % 5;
  for (int i = 0; i < in_planes; ++i) facc[i * c + co] = 0.f;
  const int b0 = chunk * per_chunk, b1 = b0 + per_chunk < n ? b0 + per_chunk : n;
  for (int b = b0; b < b1; ++b)
    for (int pix = 0; pix < 90; ++pix) {
      const int rr = pix / 9 + kh - 2, cc = pix % 9 + kw - 2;
      if (rr < 0 || rr > 9 || cc < 0 || cc > 8) continue;
      const float g = dz[((size_t)b * 90 + pix) * c + co];
      for (int h = 0; h < nb; ++h) {
        const int p = __ldg(pl + ((size_t)b * 2 + h) * 90 + rr * 9 + cc);
        if (p >= 0) facc[(h * 14 + p) * c + co] += g;
      }
    }
  for (int i = 0; i < in_planes; ++i) part[(((size_t)chunk * 25 + tap) * in_planes + i) * c + co] = facc[i * c + co];
}

// out[i] = sum_s part[s][i] in split order (scaled by *inv when given)
__global__ void k_sum_parts(const float* __restrict__ part, int splits, long long n, const float* __restrict__ inv, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += part[(size_t)k * n + i];
    out[i] = inv ? s * *inv : s;
  }
}

// wgrad partials [splits][tap][co][ci] -> Keras HWIO gradient [tap][ci][co], splits summed in order, unscaled by *inv
__global__ void k_wgrad_reduce(const float* __restrict__ part, int splits, int c, const float* __restrict__ inv, float* __restrict__ out) {
  const long long n = 9LL * c * c;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int ci = (int)(i % c), co = (int)((i / c) % c), tap = (int)(i / ((long long)c * c));
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += part[(size_t)k * n + i];
    out[((size_t)tap * c + ci) * c + co] = s * *inv;
  }
}

// master HWIO [3][3][ci][co] f32 -> forward B operand [tap][co][ci] fp16 and dgrad B operand [tap][ci][co] = W[8 - tap][ci][co]
__global__ void k_prep_conv3_train(const float* __restrict__ w, __half* __restrict__ wf, __half* __restrict__ wd, int c) {
  const long long n = 9LL * c * c;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int a = (int)(i % c), b = (int)((i / c) % c), tap = (int)(i / ((long long)c * c));
    wf[i] = __float2half_rn(w[((size_t)tap * c + a) * c + b]);          // [tap][co = b][ci = a]
    wd[i] = __float2half_rn(w[((size_t)(8 - tap) * c + b) * c + a]);    // [tap][ci = b][co = a]
  }
}

// ---- BatchNormalization, training mode --------------------------------------------------------------------------
struct BnArgs {
  const float* z; long long P; int C;
  const float *mean, *rstd, *gamma, *beta;
  const float* skip;                  // fp32 residual added before the ReLU, or null
  const float* up;                    // upstream gradient (of the ReLU output), or null (forward)
  const float* up_inv;                // device scalar multiplying `up` (unscaling of a dgrad output), or null
  int flat;                           // 1: up / forward output in Keras Flatten order [b][c*90 + pix] (heads)
};
__device__ __forceinline__ long long flat_index(const BnArgs& a, long long r, int c) {
  return a.flat ? ((r / 90) * a.C + c) * 90 + r % 90 : r * a.C + c;
}
// pre-ReLU output y = gamma * xhat + beta (+ skip); the forward's ReLU and the backward's mask both read it from here
__device__ __forceinline__ float bn_y(const BnArgs& a, long long r, int c, float& xhat) {
  xhat = (a.z[r * a.C + c] - a.mean[c]) * a.rstd[c];
  float y = __fmaf_rn(a.gamma[c], xhat, a.beta[c]);
  if (a.skip) y += a.skip[r * a.C + c];
  return y;
}
__device__ __forceinline__ float bn_g(const BnArgs& a, long long r, int c, float y) {
  if (!(y > 0.f)) return 0.f;
  const float u = a.up[flat_index(a, r, c)];
  return a.up_inv ? u * *a.up_inv : u;
}

// Per-chunk partial sums over rows, two outputs per channel: mode 0 {sum z}, 1 {sum (z - mean)^2}, 2 {sum g, sum g*xhat}.
// Thread = (lane, channel), 256 / C lanes stride the chunk's rows in order, lanes are then summed in order.
__global__ void __launch_bounds__(256) k_bn_reduce(BnArgs a, int mode, long long rows_per_chunk, float* __restrict__ part) {
  __shared__ float sh[2][256];
  const int C = a.C, lanes = 256 / C, tid = threadIdx.x, c = tid % C, lane = tid / C;
  const long long r0 = blockIdx.x * rows_per_chunk, r1 = r0 + rows_per_chunk < a.P ? r0 + rows_per_chunk : a.P;
  float s0 = 0.f, s1 = 0.f;
  if (lane < lanes) {
    for (long long r = r0 + lane; r < r1; r += lanes) {
      if (mode == 0) {
        s0 += a.z[r * C + c];
      } else if (mode == 1) {
        const float d = a.z[r * C + c] - a.mean[c];
        s0 = __fmaf_rn(d, d, s0);
      } else {
        float xhat;
        const float g = bn_g(a, r, c, bn_y(a, r, c, xhat));
        s0 += g;
        s1 = __fmaf_rn(g, xhat, s1);
      }
    }
  }
  sh[0][tid] = s0; sh[1][tid] = s1;
  __syncthreads();
  if (tid < C) {
    float t0 = 0.f, t1 = 0.f;
    for (int l = 0; l < lanes; ++l) { t0 += sh[0][l * C + c]; t1 += sh[1][l * C + c]; }
    part[((size_t)blockIdx.x * 2) * C + c] = t0;
    part[((size_t)blockIdx.x * 2 + 1) * C + c] = t1;
  }
}
// chunks summed in order.  mode 0: out0 = mean; 1: out0 = var (biased), out1 = rstd; 2: out0 = sum g, out1 = sum g*xhat
__global__ void k_bn_finalize(const float* __restrict__ part, int chunks, int C, long long P, int mode, float* out0, float* out1) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float t0 = 0.f, t1 = 0.f;
  for (int k = 0; k < chunks; ++k) { t0 += part[((size_t)k * 2) * C + c]; t1 += part[((size_t)k * 2 + 1) * C + c]; }
  if (mode == 0) out0[c] = t0 / (float)P;
  else if (mode == 1) { const float v = t0 / (float)P; out0[c] = v; out1[c] = 1.f / sqrtf(v + kBnEps); }
  else { out0[c] = t0; out1[c] = t1; }
}
// forward: out = relu(y) -> fp16 [P][C] and/or fp32 ([P][C], or the Flatten order when a.flat)
__global__ void k_bn_apply(BnArgs a, __half* __restrict__ out16, float* __restrict__ out32) {
  const long long n = a.P * a.C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / a.C;
    const int c = (int)(i % a.C);
    float xhat;
    const float o = fmaxf(bn_y(a, r, c, xhat), 0.f);
    if (out16) out16[i] = __float2half_rn(o);
    if (out32) out32[flat_index(a, r, c)] = o;
  }
}
// backward: dz = gamma * rstd * (g - sum_g / P - xhat * sum_gx / P); dz may alias a.z.  g_out (may alias a.up when not
// flat): the masked upstream gradient, i.e. the gradient reaching the skip path.  absmax: max |dz| as float bits.
__global__ void k_bn_bwd_apply(BnArgs a, const float* __restrict__ sum_g, const float* __restrict__ sum_gx, float* dz, float* g_out,
                               unsigned* absmax) {
  const long long n = a.P * a.C;
  const float invP = 1.f / (float)a.P;
  float mx = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / a.C;
    const int c = (int)(i % a.C);
    float xhat;
    const float g = bn_g(a, r, c, bn_y(a, r, c, xhat));
    const float d = a.gamma[c] * a.rstd[c] * (g - sum_g[c] * invP - xhat * (sum_gx[c] * invP));
    dz[i] = d;
    if (g_out) g_out[i] = g;
    mx = fmaxf(mx, fabsf(d));
  }
  if (absmax) {
    for (int m = 16; m; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
    if ((threadIdx.x & 31) == 0) atomicMax(absmax, __float_as_uint(mx));     // max is order-independent
  }
}
__global__ void k_absmax(const float* __restrict__ x, long long n, unsigned* absmax) {
  float mx = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) mx = fmaxf(mx, fabsf(x[i]));
  for (int m = 16; m; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
  if ((threadIdx.x & 31) == 0) atomicMax(absmax, __float_as_uint(mx));
}
// slot = {absmax bits, scale, inv}: scale = 2^e with max * scale in [2^14, 2^15) — the top of fp16's normal range with a
// factor 2 of headroom; power-of-two scaling and unscaling are exact.
__global__ void k_pick_scale(float* slot) {
  const float m = __uint_as_float(reinterpret_cast<unsigned*>(slot)[0]);
  int e = 0;
  if (m > 0.f && isfinite(m)) { e = 14 - ilogbf(m); e = e > 126 ? 126 : (e < -126 ? -126 : e); }
  slot[1] = ldexpf(1.f, e);
  slot[2] = ldexpf(1.f, -e);
}
__global__ void k_to_half_scaled(const float* __restrict__ x, long long n, const float* __restrict__ slot, __half* __restrict__ out) {
  const float s = slot[1];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = __float2half_rn(x[i] * s);
}
__global__ void k_scale(float* __restrict__ x, long long n, const float* __restrict__ s) {
  const float f = *s;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) x[i] *= f;
}
// g += d * (*inv)  (skip-path gradient + unscaled dgrad output)
__global__ void k_add_scaled(float* __restrict__ g, const float* __restrict__ d, long long n, const float* __restrict__ inv) {
  const float s = *inv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) g[i] += d[i] * s;
}

// ---- plain fp32 GEMM (heads): out[m][n] (+)= sum_k A(m, k) * B(k, n) (+ bias[n]); element (r, c) of an operand at
// p[r * sr + c * sc].  16x16 tiles, k in order; blockIdx.z = K split (partials, summed in order by k_gemm_reduce).
struct Mat { const float* p; long long sr, sc; };
__global__ void __launch_bounds__(256) k_gemm(int M, int N, int K, Mat A, Mat B, int k_per_split, float* out, long long ldo, int accumulate,
                                              const float* bias) {
  __shared__ float As[16][17], Bs[16][17];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m = blockIdx.y * 16 + ty, n = blockIdx.x * 16 + tx;
  const int k0 = blockIdx.z * k_per_split, k1 = k0 + k_per_split < K ? k0 + k_per_split : K;
  float acc = 0.f;
  for (int kt = k0; kt < k1; kt += 16) {
    const int ka = kt + tx, kb = kt + ty;
    const int am = blockIdx.y * 16 + ty, bn = blockIdx.x * 16 + tx;
    As[ty][tx] = (am < M && ka < k1) ? A.p[am * A.sr + ka * A.sc] : 0.f;
    Bs[ty][tx] = (bn < N && kb < k1) ? B.p[kb * B.sr + bn * B.sc] : 0.f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) acc = __fmaf_rn(As[ty][k], Bs[k][tx], acc);
    __syncthreads();
  }
  if (m >= M || n >= N) return;
  if (gridDim.z > 1) { out[((size_t)blockIdx.z * M + m) * N + n] = acc; return; }
  if (bias) acc += bias[n];
  float* o = out + m * ldo + n;
  *o = accumulate ? *o + acc : acc;
}
__global__ void k_gemm_reduce(const float* __restrict__ part, int splits, int M, int N, float* out, long long ldo, int accumulate,
                              const float* bias) {
  const long long n_el = (long long)M * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_el; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += part[(size_t)k * n_el + i];
    if (bias) s += bias[i % N];
    float* o = out + (i / N) * ldo + i % N;
    *o = accumulate ? *o + s : s;
  }
}

// ---- heads: losses and output gradients ------------------------------------------------------------------------
// fixed-shape block sum (256 threads): every thread's value, then a fixed tree
__device__ float block_sum(float v, float* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = 128; s; s >>= 1) { if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s]; __syncthreads(); }
  const float r = red[0];
  __syncthreads();
  return r;
}
__device__ float block_max(float v, float* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = 128; s; s >>= 1) { if ((int)threadIdx.x < s) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + s]); __syncthreads(); }
  const float r = red[0];
  __syncthreads();
  return r;
}
// Keras categorical_crossentropy on a softmax output (TF backend): p^ = p / sum p, clipped to [eps, 1 - eps] (eps = 1e-7 in
// fp32), loss = -sum t log p^.  A target term whose p^ lies outside the interval has zero gradient.  grid = batch, block = 256.
// dlog = w_p / n * dloss / dlogits.
__global__ void __launch_bounds__(256) k_policy_loss(const float* __restrict__ logits, const float* __restrict__ target, int n, float w_p,
                                                     float* __restrict__ dlog, float* __restrict__ ce_rows) {
  __shared__ float p[kLabels];
  __shared__ float red[256];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* l = logits + (size_t)b * kLabels;
  const float* t = target + (size_t)b * kLabels;
  const float eps = 1e-7f, hi = 1.f - eps;
  float mx = -INFINITY;
  for (int j = tid; j < kLabels; j += 256) mx = fmaxf(mx, l[j]);
  mx = block_max(mx, red);
  float s = 0.f;
  for (int j = tid; j < kLabels; j += 256) { p[j] = expf(l[j] - mx); s += p[j]; }
  const float inv = 1.f / block_sum(s, red);
  float S = 0.f;
  for (int j = tid; j < kLabels; j += 256) { p[j] *= inv; S += p[j]; }
  S = block_sum(S, red);
  float loss = 0.f, A = 0.f;
  for (int j = tid; j < kLabels; j += 256) {
    const float ph = p[j] / S, tj = t[j];
    const float c = fminf(fmaxf(ph, eps), hi);
    if (tj != 0.f) loss -= tj * logf(c);
    const float u = (ph >= eps && ph <= hi && tj != 0.f) ? -tj / c : 0.f;
    A += u * ph;
  }
  loss = block_sum(loss, red);
  A = block_sum(A, red);
  float Bs = 0.f;
  for (int j = tid; j < kLabels; j += 256) {
    const float ph = p[j] / S, tj = t[j];
    const float c = fminf(fmaxf(ph, eps), hi);
    const float u = (ph >= eps && ph <= hi && tj != 0.f) ? -tj / c : 0.f;
    const float g = (u - A) / S;
    Bs += g * p[j];
  }
  Bs = block_sum(Bs, red);
  const float scale = w_p / (float)n;
  for (int j = tid; j < kLabels; j += 256) {
    const float ph = p[j] / S, tj = t[j];
    const float c = fminf(fmaxf(ph, eps), hi);
    const float u = (ph >= eps && ph <= hi && tj != 0.f) ? -tj / c : 0.f;
    dlog[(size_t)b * kLabels + j] = p[j] * ((u - A) / S - Bs) * scale;
  }
  if (tid == 0) ce_rows[b] = loss;
}
// value = tanh(pre); squared error per row; dpre = w_v * 2 (v - z) / n * (1 - v^2)
__global__ void k_value_loss(const float* __restrict__ pre, const float* __restrict__ z, int n, float w_v, float* __restrict__ se_rows,
                             float* __restrict__ dpre) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n) return;
  const float v = tanhf(pre[b]), d = v - z[b];
  se_rows[b] = d * d;
  dpre[b] = w_v * 2.f * d / (float)n * (1.f - v * v);
}
__global__ void k_relu_mask(const float* __restrict__ pre, float* __restrict__ out, float* __restrict__ grad, long long n) {
  // out = relu(pre) when grad == null (forward); grad *= (pre > 0) otherwise
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (grad) { if (!(pre[i] > 0.f)) grad[i] = 0.f; }
    else out[i] = fmaxf(pre[i], 0.f);
  }
}
// one block: sum of squares of a tensor (fixed order) -> slot
__global__ void __launch_bounds__(256) k_sumsq(const float* __restrict__ x, long long n, float* slot) {
  __shared__ float red[256];
  float s = 0.f;
  for (long long i = threadIdx.x; i < n; i += 256) s = __fmaf_rn(x[i], x[i], s);
  s = block_sum(s, red);
  if (threadIdx.x == 0) *slot = s;
}
// losses = {total, policy CE, value MSE, l2}
__global__ void __launch_bounds__(256) k_losses(const float* __restrict__ ce, const float* __restrict__ se, int n, const float* __restrict__ l2_slots,
                                                int n_slots, float l2, float w_p, float w_v, float* losses) {
  __shared__ float red[256];
  float a = 0.f, b = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) { a += ce[i]; b += se[i]; }
  a = block_sum(a, red) / (float)n;
  b = block_sum(b, red) / (float)n;
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < n_slots; ++i) s += l2_slots[i];
    const float l = l2 * s;
    losses[0] = w_p * a + w_v * b + l; losses[1] = a; losses[2] = b; losses[3] = l;
  }
}
// Keras SGD (momentum, no Nesterov, decay 0): v = mu * v - lr * (g + 2 * l2 * w); w = w + v
__global__ void k_sgd(float* __restrict__ w, float* __restrict__ v, const float* __restrict__ g, long long n, float lr, float mu, float l2x2) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gt = g[i] + l2x2 * w[i];
    const float vn = mu * v[i] - lr * gt;
    v[i] = vn;
    w[i] += vn;
  }
}
// Keras 2.0.8 Adam (decay 0), every trainable tensor in ONE launch: block b updates chunk b - block0 of the segment that
// owns it.  The operations are spelled out (no contraction) so that a float32 restatement in the same order is bit-exact:
//   g = grad + 2*l2*w (kernels);  m = b1*m + (1-b1)*g;  v = b2*v + (1-b2)*g*g;  w = w - (lr_t*m) / (sqrt(v) + eps)
constexpr int kAdamChunk = 2048;
struct AdamSeg { float* w; float* m; float* v; const float* g; long long n; long long block0; int reg; int pad; };
__global__ void k_adam(const AdamSeg* __restrict__ seg, int nseg, float lr_t, float b1, float omb1, float b2, float omb2, float eps,
                       float l2x2) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (seg[mid].block0 <= (long long)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const AdamSeg s = seg[lo];
  const long long base = ((long long)blockIdx.x - s.block0) * kAdamChunk;
  const long long end = base + kAdamChunk < s.n ? base + kAdamChunk : s.n;
  for (long long i = base + threadIdx.x; i < end; i += blockDim.x) {
    const float w = s.w[i];
    const float g = s.reg ? __fadd_rn(s.g[i], __fmul_rn(l2x2, w)) : s.g[i];
    const float m = __fadd_rn(__fmul_rn(b1, s.m[i]), __fmul_rn(omb1, g));
    const float v = __fadd_rn(__fmul_rn(b2, s.v[i]), __fmul_rn(omb2, __fmul_rn(g, g)));
    s.m[i] = m;
    s.v[i] = v;
    s.w[i] = __fsub_rn(w, __fdiv_rn(__fmul_rn(lr_t, m), __fadd_rn(__fsqrt_rn(v), eps)));
  }
}
// Keras moving_average_update (TF assign_moving_average, zero_debias off): m -= (m - batch) * (1 - 0.99)
__global__ void k_moving(float* __restrict__ m, const float* __restrict__ batch, int c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < c) m[i] -= (m[i] - batch[i]) * (1.f - 0.99f);
}
__global__ void k_fill(float* p, long long n, float v) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

// ------------------------------------------------------------------------------------------------ host side
struct Param {
  std::string layer, weight;   // Keras layer prefix ("res3_conv1") and weight ("kernel")
  long long numel;
  bool train, reg;             // updated by SGD / carries the L2 penalty (kernels)
  float *w, *v, *g;            // master (caller), velocity (caller), gradient (workspace)
  float *am, *av;              // Adam moments (caller), set by cz_train_set_adam
};
struct Bn {
  int C; int gamma, beta, mm, mv;   // Param indices
  float* z;                          // pre-BN input [P][C]; the backward writes dz over it
  float *mean, *var, *rstd;          // batch statistics of the last step
};

struct Trainer {
  cz_train_config cfg;
  int C, L, ip, pc, vc, H, maxb;
  cudaStream_t st;
  std::vector<Param> p;
  std::vector<Bn> bn;                // 0 = input, 1 + 2i + j = block i conv j + 1, then policy, value
  int i_first, i_pol_k, i_pol_dense_k, i_pol_dense_b, i_val_k, i_vd_k, i_vd_b, i_vo_k, i_vo_b;
  std::vector<int> i_conv;          // [2L] kernel indices
  bool params_set;
  int last_batch;
  // workspace
  int8_t* pl;
  std::vector<__half*> a16, h16;     // [L + 1] block inputs / outputs, [L] conv1 outputs (fp16, conv inputs)
  std::vector<float*> s32;           // [L + 1] the same block outputs in fp32 (skip stream, heads input)
  float *G, *D; __half* dz16;
  std::vector<__half*> wf16, wd16;   // [2L] forward / dgrad operands
  std::vector<CUtensorMap> map_wf, map_wd;
  std::vector<CUtensorMap> hm_a, hm_h, im_a64, im_h64;   // conv inputs: halo maps (forward convs), im2col maps (wgrad)
  CUtensorMap hm_dz, map_dz;
  float* wg_part; float* fw_part; float* col_part; float* gemm_part;
  float* scale_slots;                // [2L + 1][4]
  float *Fp, *Fv, *logits, *dlog, *hpre, *hact, *vpre, *dvpre, *dh, *dF, *ce_rows, *se_rows, *ones;
  float* l2_slots; int n_reg;
  // Adam (cz_train_set_adam): the segment table lives in the workspace
  bool adam;
  double b1, b2, eps;
  long long iterations;
  AdamSeg* adam_tab; int n_adam; long long adam_blocks;
  std::vector<AdamSeg> adam_host;
};

static size_t act_bytes(const Trainer* t, int elem) { return (size_t)t->maxb * 90 * t->C * elem; }

static void layout(Trainer* t, Carver& cv) {
  const int C = t->C, L = t->L, B = t->maxb;
  const size_t P = (size_t)B * 90;
  t->pl = (int8_t*)cv.take((size_t)B * 2 * 90);
  t->a16.assign(L + 1, nullptr); t->s32.assign(L + 1, nullptr); t->h16.assign(L, nullptr);
  for (int k = 0; k <= L; ++k) { t->a16[k] = (__half*)cv.take(act_bytes(t, 2)); t->s32[k] = (float*)cv.take(act_bytes(t, 4)); }
  for (int k = 0; k < L; ++k) t->h16[k] = (__half*)cv.take(act_bytes(t, 2));
  for (Bn& b : t->bn) {
    b.z = (float*)cv.take(P * b.C * 4);
    b.mean = (float*)cv.take(b.C * 4); b.var = (float*)cv.take(b.C * 4); b.rstd = (float*)cv.take(b.C * 4);
  }
  t->G = (float*)cv.take(act_bytes(t, 4));
  t->D = (float*)cv.take(act_bytes(t, 4));
  t->dz16 = (__half*)cv.take(act_bytes(t, 2));
  t->wf16.assign(2 * L, nullptr); t->wd16.assign(2 * L, nullptr);
  for (int l = 0; l < 2 * L; ++l) { t->wf16[l] = (__half*)cv.take(9ULL * C * C * 2); t->wd16[l] = (__half*)cv.take(9ULL * C * C * 2); }
  t->wg_part = (float*)cv.take((size_t)kMaxSplits * 9 * C * C * 4);
  t->fw_part = (float*)cv.take((size_t)16 * 25 * t->ip * C * 4);
  t->col_part = (float*)cv.take((size_t)1024 * 2 * 256 * 4);
  t->gemm_part = (float*)cv.take((size_t)kGemmPartFloats * 4);
  t->scale_slots = (float*)cv.take((size_t)(2 * L + 1) * 4 * 4);
  const int pk = t->pc * 90, vk = t->vc * 90;
  t->Fp = (float*)cv.take((size_t)B * pk * 4);
  t->Fv = (float*)cv.take((size_t)B * vk * 4);
  t->logits = (float*)cv.take((size_t)B * kLabels * 4);
  t->dlog = (float*)cv.take((size_t)B * kLabels * 4);
  t->hpre = (float*)cv.take((size_t)B * t->H * 4);
  t->hact = (float*)cv.take((size_t)B * t->H * 4);
  t->dh = (float*)cv.take((size_t)B * t->H * 4);
  t->vpre = (float*)cv.take((size_t)B * 4);
  t->dvpre = (float*)cv.take((size_t)B * 4);
  t->dF = (float*)cv.take((size_t)B * (pk > vk ? pk : vk) * 4);
  t->ce_rows = (float*)cv.take((size_t)B * 4);
  t->se_rows = (float*)cv.take((size_t)B * 4);
  t->ones = (float*)cv.take((size_t)B * 4);
  t->l2_slots = (float*)cv.take((size_t)(t->p.size() + 1) * 4);
  for (Param& q : t->p) q.g = (float*)cv.take((size_t)q.numel * 4);
  t->adam_tab = (AdamSeg*)cv.take(t->p.size() * sizeof(AdamSeg));
}

static void add_bn(Trainer* t, const std::string& layer, int c) {
  Bn b; memset(&b, 0, sizeof(b));
  b.C = c;
  const char* names[4] = {"gamma", "beta", "moving_mean", "moving_variance"};
  int* idx[4] = {&b.gamma, &b.beta, &b.mm, &b.mv};
  for (int k = 0; k < 4; ++k) {
    *idx[k] = (int)t->p.size();
    t->p.push_back(Param{layer, names[k], c, k < 2, false, nullptr, nullptr, nullptr});
  }
  t->bn.push_back(b);
}
static int add_param(Trainer* t, const std::string& layer, const std::string& weight, long long numel, bool reg) {
  t->p.push_back(Param{layer, weight, numel, true, reg, nullptr, nullptr, nullptr});
  return (int)t->p.size() - 1;
}

static void describe(Trainer* t) {
  const int C = t->C;
  t->p.clear(); t->bn.clear(); t->i_conv.clear();
  t->i_first = add_param(t, "input_conv", "kernel", 25LL * t->ip * C, true);
  add_bn(t, "input_batchnorm", C);
  for (int i = 0; i < t->L; ++i)
    for (int j = 0; j < 2; ++j) {
      t->i_conv.push_back(add_param(t, "res" + std::to_string(i + 1) + "_conv" + std::to_string(j + 1), "kernel", 9LL * C * C, true));
      add_bn(t, "res" + std::to_string(i + 1) + "_batchnorm" + std::to_string(j + 1), C);
    }
  t->i_pol_k = add_param(t, "policy_conv", "kernel", (long long)C * t->pc, true);
  add_bn(t, "policy_batchnorm", t->pc);
  t->i_pol_dense_k = add_param(t, "policy_out", "kernel", 90LL * t->pc * kLabels, true);
  t->i_pol_dense_b = add_param(t, "policy_out", "bias", kLabels, false);
  t->i_val_k = add_param(t, "value_conv", "kernel", (long long)C * t->vc, true);
  add_bn(t, "value_batchnorm", t->vc);
  t->i_vd_k = add_param(t, "value_dense", "kernel", 90LL * t->vc * t->H, true);
  t->i_vd_b = add_param(t, "value_dense", "bias", t->H, false);
  t->i_vo_k = add_param(t, "value_out", "kernel", t->H, true);
  t->i_vo_b = add_param(t, "value_out", "bias", 1, false);
  t->n_reg = 0;
  for (const Param& q : t->p) t->n_reg += q.reg ? 1 : 0;
}

static int check_cfg(const cz_train_config* c) {
  if (!c || c->struct_bytes != (int)sizeof(cz_train_config)) return cz_fail(CZ_ERR_ARG, "cz_train: config struct_bytes mismatch");
  if (c->filters < 64 || c->filters > 256 || c->filters % 64) return cz_fail(CZ_ERR_UNSUPPORTED, "cz_train: filters must be 64..256 step 64");
  if (c->blocks < 0 || c->blocks > 64) return cz_fail(CZ_ERR_ARG, "cz_train: blocks %d", c->blocks);
  if (c->in_planes != 14 && c->in_planes != 28) return cz_fail(CZ_ERR_UNSUPPORTED, "cz_train: 14 or 28 input planes");
  if (c->policy_channels < 1 || c->policy_channels > 32 || c->value_channels < 1 || c->value_channels > 4)
    return cz_fail(CZ_ERR_UNSUPPORTED, "cz_train: head widths up to 32 policy / 4 value channels");
  if (c->value_fc < 1 || c->value_fc > 256) return cz_fail(CZ_ERR_UNSUPPORTED, "cz_train: value_fc must be 1..256");
  if (c->max_batch < 1 || c->max_batch > 4096) return cz_fail(CZ_ERR_ARG, "cz_train: max_batch must be 1..4096");
  return 0;
}
static void init_geometry(Trainer* t, const cz_train_config* c) {
  t->cfg = *c;
  t->C = c->filters; t->L = c->blocks; t->ip = c->in_planes; t->pc = c->policy_channels; t->vc = c->value_channels;
  t->H = c->value_fc; t->maxb = c->max_batch;
  describe(t);
}

// ---- launch helpers
static int gemm(Trainer* t, int M, int N, int K, Mat A, Mat B, float* out, long long ldo, int accumulate, const float* bias) {
  const int tiles = ((M + 15) / 16) * ((N + 15) / 16);
  int splits = 1;
  if (tiles < 264 && K >= 2048) {
    splits = 528 / tiles;
    if (splits > K / 256) splits = K / 256;
    if (splits > kGemmMaxSplits) splits = kGemmMaxSplits;
    if ((long long)splits * M * N > kGemmPartFloats) splits = (int)(kGemmPartFloats / ((long long)M * N));
    if (splits < 1) splits = 1;
  }
  const int kps = ((K + splits - 1) / splits + 15) / 16 * 16;
  splits = (K + kps - 1) / kps;
  dim3 grid((N + 15) / 16, (M + 15) / 16, splits);
  if (splits > 1) {
    k_gemm<<<grid, 256, 0, t->st>>>(M, N, K, A, B, kps, t->gemm_part, N, 0, nullptr);
    k_gemm_reduce<<<blocks_for((long long)M * N), 256, 0, t->st>>>(t->gemm_part, splits, M, N, out, ldo, accumulate, bias);
  } else {
    k_gemm<<<grid, 256, 0, t->st>>>(M, N, K, A, B, kps, out, ldo, accumulate, bias);
  }
  CZ_CUDA(cudaGetLastError());
  return 0;
}

static int col_chunks(long long P, long long* rows) {
  long long ch = (P + 63) / 64;
  if (ch > 1024) ch = 1024;
  *rows = (P + ch - 1) / ch;
  return (int)((P + *rows - 1) / *rows);
}
static BnArgs bn_args(Trainer* t, const Bn& b, long long P, const float* skip) {
  BnArgs a; memset(&a, 0, sizeof(a));
  a.z = b.z; a.P = P; a.C = b.C; a.mean = b.mean; a.rstd = b.rstd;
  a.gamma = t->p[b.gamma].w; a.beta = t->p[b.beta].w; a.skip = skip;
  return a;
}
// batch statistics (two passes) then relu(BN(z) (+ skip)) -> out16 / out32
static int bn_forward(Trainer* t, Bn& b, long long P, const float* skip, __half* out16, float* out32, int flat) {
  long long rows;
  const int ch = col_chunks(P, &rows);
  BnArgs a = bn_args(t, b, P, skip);
  k_bn_reduce<<<ch, 256, 0, t->st>>>(a, 0, rows, t->col_part);
  k_bn_finalize<<<1, 256, 0, t->st>>>(t->col_part, ch, b.C, P, 0, b.mean, nullptr);
  k_bn_reduce<<<ch, 256, 0, t->st>>>(a, 1, rows, t->col_part);
  k_bn_finalize<<<1, 256, 0, t->st>>>(t->col_part, ch, b.C, P, 1, b.var, b.rstd);
  a.flat = flat;
  k_bn_apply<<<blocks_for(P * b.C), 256, 0, t->st>>>(a, out16, out32);
  CZ_CUDA(cudaGetLastError());
  return 0;
}
// BN backward from the upstream gradient of the ReLU output: dgamma / dbeta into the gradient buffers, dz over b.z;
// g_out = masked upstream (skip path); scale slot gets max |dz| when given
static int bn_backward(Trainer* t, Bn& b, long long P, const float* skip, const float* up, const float* up_inv, int flat, float* g_out,
                       float* slot) {
  long long rows;
  const int ch = col_chunks(P, &rows);
  BnArgs a = bn_args(t, b, P, skip);
  a.up = up; a.up_inv = up_inv; a.flat = flat;
  float *dbeta = t->p[b.beta].g, *dgamma = t->p[b.gamma].g;
  k_bn_reduce<<<ch, 256, 0, t->st>>>(a, 2, rows, t->col_part);
  k_bn_finalize<<<1, 256, 0, t->st>>>(t->col_part, ch, b.C, P, 2, dbeta, dgamma);
  if (slot) CZ_CUDA(cudaMemsetAsync(slot, 0, 4, t->st));
  k_bn_bwd_apply<<<blocks_for(P * b.C), 256, 0, t->st>>>(a, dbeta, dgamma, b.z, g_out, slot ? reinterpret_cast<unsigned*>(slot) : nullptr);
  CZ_CUDA(cudaGetLastError());
  return 0;
}

// raw fp32 3x3 conv of fp16 activations (halo map `in`) with fp16 weights (map boxes of conv_tile_n rows)
static int conv3x3(int n, int c, const CUtensorMap& in, const CUtensorMap& w, float* out, cudaStream_t st) {
  igemm::Args a = cznn::conv_args(n, c, nullptr, nullptr, out, 0);
  a.out_f32 = 1;
  return cznn::launch_igemm(cznn::conv_tile_n(c, false), in, w, a, st);
}

template <int NB>
static int launch_wgrad_t(const CUtensorMap& dy, const CUtensorMap& x, const wgrad::Args& a, cudaStream_t st) {
  using Cf = wgrad::Cfg<NB>;
  static bool attr = false;
  if (!attr) { CZ_CUDA(cudaFuncSetAttribute(wgrad::k_wgrad<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cf::kSmemBytes)); attr = true; }
  wgrad::k_wgrad<NB><<<9 * a.co_tiles * a.splits, wgrad::kThreads, Cf::kSmemBytes, st>>>(dy, x, a);
  CZ_CUDA(cudaGetLastError());
  return 0;
}
// dW (Keras HWIO, fp32) = wgrad(dy16 scaled by slot[1], x16) * slot[2]
static int wgrad_launch(int c, int n, const CUtensorMap& dy, const CUtensorMap& x, float* part, const float* slot, float* out, cudaStream_t st) {
  wgrad::Args a;
  a.c = c; a.co_tiles = (c + 127) / 128; a.chunks = (n * 90 + wgrad::kPix - 1) / wgrad::kPix; a.part = part;
  int splits = cznn::num_sms() / (9 * a.co_tiles);
  if (splits > kMaxSplits) splits = kMaxSplits;
  if (splits > a.chunks) splits = a.chunks;
  if (splits < 1) splits = 1;
  const int per = (a.chunks + splits - 1) / splits;
  a.splits = (a.chunks + per - 1) / per;              // every split gets at least one chunk
  int rc = 0;
  switch (c / 64) {
    case 1: rc = launch_wgrad_t<1>(dy, x, a, st); break;
    case 2: rc = launch_wgrad_t<2>(dy, x, a, st); break;
    case 3: rc = launch_wgrad_t<3>(dy, x, a, st); break;
    case 4: rc = launch_wgrad_t<4>(dy, x, a, st); break;
    default: return cz_fail(CZ_ERR_UNSUPPORTED, "wgrad: filters must be 64..256 step 64");
  }
  if (rc) return rc;
  k_wgrad_reduce<<<blocks_for(9LL * c * c), 256, 0, st>>>(part, a.splits, c, slot + 2, out);
  CZ_CUDA(cudaGetLastError());
  return 0;
}

static int build_maps(Trainer* t, int n) {
  if (t->last_batch == n) return 0;
  const int C = t->C, L = t->L;
  const long long P = (long long)n * 90;
  t->hm_a.resize(L + 1); t->im_a64.resize(L + 1); t->hm_h.resize(L); t->im_h64.resize(L);
  for (int k = 0; k <= L; ++k) {
    CZ_TRY(cznn::make_map_2d(&t->hm_a[k], t->a16[k], C, P, igemm::kHaloBox));
    CZ_TRY(cznn::make_map_im2col(&t->im_a64[k], t->a16[k], C, n, wgrad::kPix));
  }
  for (int k = 0; k < L; ++k) {
    CZ_TRY(cznn::make_map_2d(&t->hm_h[k], t->h16[k], C, P, igemm::kHaloBox));
    CZ_TRY(cznn::make_map_im2col(&t->im_h64[k], t->h16[k], C, n, wgrad::kPix));
  }
  CZ_TRY(cznn::make_map_2d(&t->hm_dz, t->dz16, C, P, igemm::kHaloBox));
  CZ_TRY(cznn::make_map_2d(&t->map_dz, t->dz16, C, (long long)n * 90, wgrad::kPix));
  t->last_batch = n;
  return 0;
}

// ---- the step
static int step(Trainer* t, const float* planes, const float* pol_t, const float* val_t, int n, const cz_train_hparams& hp, float* losses) {
  const int C = t->C, L = t->L, pc = t->pc, vc = t->vc, H = t->H;
  const long long P = (long long)n * 90, PC = P * C;
  cudaStream_t st = t->st;
  CZ_TRY(build_maps(t, n));
  // operands of the tensor-core convolutions from the master weights
  for (int l = 0; l < 2 * L; ++l)
    k_prep_conv3_train<<<blocks_for(9LL * C * C), 256, 0, st>>>(t->p[t->i_conv[l]].w, t->wf16[l], t->wd16[l], C);
  // ---------------------------------------------------------------- forward
  k_plane_index<<<blocks_for((long long)n * (t->ip / 14) * 90), 256, 0, st>>>(planes, t->pl, n, t->ip);
  k_first_fwd<<<n, C, 0, st>>>(t->pl, t->p[t->i_first].w, t->bn[0].z, C, t->ip);
  CZ_TRY(bn_forward(t, t->bn[0], P, nullptr, t->a16[0], t->s32[0], 0));
  for (int i = 0; i < L; ++i) {
    Bn &b1 = t->bn[1 + 2 * i], &b2 = t->bn[2 + 2 * i];
    CZ_TRY(conv3x3(n, C, t->hm_a[i], t->map_wf[2 * i], b1.z, st));
    CZ_TRY(bn_forward(t, b1, P, nullptr, t->h16[i], nullptr, 0));
    CZ_TRY(conv3x3(n, C, t->hm_h[i], t->map_wf[2 * i + 1], b2.z, st));
    CZ_TRY(bn_forward(t, b2, P, t->s32[i], t->a16[i + 1], t->s32[i + 1], 0));
  }
  const float* S = t->s32[L];
  Bn &bp = t->bn[1 + 2 * L], &bv = t->bn[2 + 2 * L];
  const Param &Wp = t->p[t->i_pol_k], &Wd = t->p[t->i_pol_dense_k], &bd = t->p[t->i_pol_dense_b];
  const Param &Wv = t->p[t->i_val_k], &W1 = t->p[t->i_vd_k], &b1 = t->p[t->i_vd_b], &W2 = t->p[t->i_vo_k], &b2 = t->p[t->i_vo_b];
  const int pk = pc * 90, vk = vc * 90;
  CZ_TRY(gemm(t, (int)P, pc, C, Mat{S, C, 1}, Mat{Wp.w, pc, 1}, bp.z, pc, 0, nullptr));
  CZ_TRY(bn_forward(t, bp, P, nullptr, nullptr, t->Fp, 1));
  CZ_TRY(gemm(t, n, kLabels, pk, Mat{t->Fp, pk, 1}, Mat{Wd.w, kLabels, 1}, t->logits, kLabels, 0, bd.w));
  CZ_TRY(gemm(t, (int)P, vc, C, Mat{S, C, 1}, Mat{Wv.w, vc, 1}, bv.z, vc, 0, nullptr));
  CZ_TRY(bn_forward(t, bv, P, nullptr, nullptr, t->Fv, 1));
  CZ_TRY(gemm(t, n, H, vk, Mat{t->Fv, vk, 1}, Mat{W1.w, H, 1}, t->hpre, H, 0, b1.w));
  k_relu_mask<<<blocks_for((long long)n * H), 256, 0, st>>>(t->hpre, t->hact, nullptr, (long long)n * H);
  CZ_TRY(gemm(t, n, 1, H, Mat{t->hact, H, 1}, Mat{W2.w, 1, 1}, t->vpre, 1, 0, b2.w));
  // ---------------------------------------------------------------- losses and output gradients
  k_policy_loss<<<n, 256, 0, st>>>(t->logits, pol_t, n, hp.w_policy, t->dlog, t->ce_rows);
  k_value_loss<<<(n + 255) / 256, 256, 0, st>>>(t->vpre, val_t, n, hp.w_value, t->se_rows, t->dvpre);
  // ---------------------------------------------------------------- heads backward
  CZ_TRY(gemm(t, H, 1, n, Mat{t->hact, 1, H}, Mat{t->dvpre, 1, 1}, W2.g, 1, 0, nullptr));          // dW2 = h^T dv
  CZ_TRY(gemm(t, 1, 1, n, Mat{t->ones, 0, 1}, Mat{t->dvpre, 1, 1}, b2.g, 1, 0, nullptr));           // db2
  CZ_TRY(gemm(t, n, H, 1, Mat{t->dvpre, 1, 1}, Mat{W2.w, 1, 1}, t->dh, H, 0, nullptr));             // dh = dv W2^T
  k_relu_mask<<<blocks_for((long long)n * H), 256, 0, st>>>(t->hpre, nullptr, t->dh, (long long)n * H);
  CZ_TRY(gemm(t, vk, H, n, Mat{t->Fv, 1, vk}, Mat{t->dh, H, 1}, W1.g, H, 0, nullptr));              // dW1 = Fv^T dh
  CZ_TRY(gemm(t, 1, H, n, Mat{t->ones, 0, 1}, Mat{t->dh, H, 1}, b1.g, H, 0, nullptr));              // db1
  CZ_TRY(gemm(t, n, vk, H, Mat{t->dh, H, 1}, Mat{W1.w, 1, H}, t->dF, vk, 0, nullptr));              // dFv = dh W1^T
  CZ_TRY(bn_backward(t, bv, P, nullptr, t->dF, nullptr, 1, nullptr, nullptr));                      // dzv over bv.z
  CZ_TRY(gemm(t, pk, kLabels, n, Mat{t->Fp, 1, pk}, Mat{t->dlog, kLabels, 1}, Wd.g, kLabels, 0, nullptr));   // dWd
  CZ_TRY(gemm(t, 1, kLabels, n, Mat{t->ones, 0, 1}, Mat{t->dlog, kLabels, 1}, bd.g, kLabels, 0, nullptr));   // dbd
  CZ_TRY(gemm(t, n, pk, kLabels, Mat{t->dlog, kLabels, 1}, Mat{Wd.w, 1, kLabels}, t->dF, pk, 0, nullptr));   // dFp
  CZ_TRY(bn_backward(t, bp, P, nullptr, t->dF, nullptr, 1, nullptr, nullptr));                      // dzp over bp.z
  CZ_TRY(gemm(t, C, pc, (int)P, Mat{S, 1, C}, Mat{bp.z, pc, 1}, Wp.g, pc, 0, nullptr));             // dWp = S^T dzp
  CZ_TRY(gemm(t, C, vc, (int)P, Mat{S, 1, C}, Mat{bv.z, vc, 1}, Wv.g, vc, 0, nullptr));             // dWv
  CZ_TRY(gemm(t, (int)P, C, pc, Mat{bp.z, pc, 1}, Mat{Wp.w, 1, pc}, t->G, C, 0, nullptr));          // G = dzp Wp^T
  CZ_TRY(gemm(t, (int)P, C, vc, Mat{bv.z, vc, 1}, Mat{Wv.w, 1, vc}, t->G, C, 1, nullptr));          //   + dzv Wv^T
  // ---------------------------------------------------------------- tower backward
  for (int i = L - 1; i >= 0; --i) {
    Bn &c1 = t->bn[1 + 2 * i], &c2 = t->bn[2 + 2 * i];
    float *slot2 = t->scale_slots + 4 * (2 * i + 1), *slot1 = t->scale_slots + 4 * (2 * i);
    // conv2: G (gradient of the block output) -> dz2, G <- masked G (the skip path)
    CZ_TRY(bn_backward(t, c2, P, t->s32[i], t->G, nullptr, 0, t->G, slot2));
    k_pick_scale<<<1, 1, 0, st>>>(slot2);
    k_to_half_scaled<<<blocks_for(PC), 256, 0, st>>>(c2.z, PC, slot2, t->dz16);
    CZ_TRY(wgrad_launch(C, n, t->map_dz, t->im_h64[i], t->wg_part, slot2, t->p[t->i_conv[2 * i + 1]].g, st));
    CZ_TRY(conv3x3(n, C, t->hm_dz, t->map_wd[2 * i + 1], t->D, st));
    // conv1: D * inv2 (gradient of the conv1 activation) -> dz1
    CZ_TRY(bn_backward(t, c1, P, nullptr, t->D, slot2 + 2, 0, nullptr, slot1));
    k_pick_scale<<<1, 1, 0, st>>>(slot1);
    k_to_half_scaled<<<blocks_for(PC), 256, 0, st>>>(c1.z, PC, slot1, t->dz16);
    CZ_TRY(wgrad_launch(C, n, t->map_dz, t->im_a64[i], t->wg_part, slot1, t->p[t->i_conv[2 * i]].g, st));
    CZ_TRY(conv3x3(n, C, t->hm_dz, t->map_wd[2 * i], t->D, st));
    k_add_scaled<<<blocks_for(PC), 256, 0, st>>>(t->G, t->D, PC, slot1 + 2);
  }
  CZ_TRY(bn_backward(t, t->bn[0], P, nullptr, t->G, nullptr, 0, nullptr, nullptr));
  {
    int chunks = (n + 63) / 64;
    if (chunks > 16) chunks = 16;
    const int per = (n + chunks - 1) / chunks;
    chunks = (n + per - 1) / per;
    k_first_wgrad<<<dim3(25, chunks), C, (size_t)t->ip * C * 4, st>>>(t->pl, t->bn[0].z, t->fw_part, n, per, C, t->ip);
    const long long nel = 25LL * t->ip * C;
    k_sum_parts<<<blocks_for(nel), 256, 0, st>>>(t->fw_part, chunks, nel, nullptr, t->p[t->i_first].g);
  }
  // ---------------------------------------------------------------- losses (L2 on the weights before the update)
  int slot = 0;
  for (const Param& q : t->p)
    if (q.reg) k_sumsq<<<1, 256, 0, st>>>(q.w, q.numel, t->l2_slots + slot++);
  k_losses<<<1, 256, 0, st>>>(t->ce_rows, t->se_rows, n, t->l2_slots, slot, hp.l2, hp.w_policy, hp.w_value, losses);
  // ---------------------------------------------------------------- update
  if (t->adam) {
    // lr_t = lr * (sqrt(1 - b2^t) / (1 - b1^t)), t = iterations + 1: float64 on the host, rounded to fp32 once
    const double it = (double)(t->iterations + 1);
    const float lr_t = (float)((double)hp.lr * (sqrt(1.0 - pow(t->b2, it)) / (1.0 - pow(t->b1, it))));
    const float b1 = (float)t->b1, b2 = (float)t->b2;
    k_adam<<<(unsigned)t->adam_blocks, 256, 0, st>>>(t->adam_tab, t->n_adam, lr_t, b1, 1.f - b1, b2, 1.f - b2, (float)t->eps,
                                                      2.f * hp.l2);
  } else {
    for (const Param& q : t->p)
      if (q.train) k_sgd<<<blocks_for(q.numel), 256, 0, st>>>(q.w, q.v, q.g, q.numel, hp.lr, hp.momentum, q.reg ? 2.f * hp.l2 : 0.f);
  }
  for (const Bn& b : t->bn) {
    k_moving<<<(b.C + 255) / 256, 256, 0, st>>>(t->p[b.mm].w, b.mean, b.C);
    k_moving<<<(b.C + 255) / 256, 256, 0, st>>>(t->p[b.mv].w, b.var, b.C);
  }
  CZ_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cztrain

// ------------------------------------------------------------------------------------------------ C ABI
struct cz_trainer { cztrain::Trainer t; };

extern "C" {
using namespace cztrain;

int cz_train_workspace_bytes(const cz_train_config* cfg, uint64_t* bytes) {
  CZ_TRY(check_cfg(cfg));
  if (!bytes) return cz_fail(CZ_ERR_ARG, "cz_train_workspace_bytes: null output");
  Trainer t;
  init_geometry(&t, cfg);
  Carver cv{nullptr, 0};
  layout(&t, cv);
  *bytes = cv.off + 4096;
  return 0;
}

int cz_train_create(const cz_train_config* cfg, void* workspace, uint64_t bytes, void* stream, cz_trainer** out) {
  CZ_TRY(check_cfg(cfg));
  if (!out || !workspace) return cz_fail(CZ_ERR_ARG, "cz_train_create: null workspace or output");
  uint64_t need = 0;
  CZ_TRY(cz_train_workspace_bytes(cfg, &need));
  if (bytes < need) return cz_fail(CZ_ERR_ARG, "cz_train_create: workspace %llu bytes < %llu", (unsigned long long)bytes, (unsigned long long)need);
  cz_trainer* h = new cz_trainer();
  Trainer* t = &h->t;
  init_geometry(t, cfg);
  t->st = (cudaStream_t)stream;
  t->params_set = false; t->last_batch = -1;
  t->adam = false; t->iterations = 0; t->n_adam = 0; t->adam_blocks = 0;
  Carver cv{(uint8_t*)workspace, 0};
  layout(t, cv);
  const int C = t->C;
  t->map_wf.resize(2 * t->L); t->map_wd.resize(2 * t->L);
  int rc = 0;
  for (int l = 0; l < 2 * t->L && !rc; ++l) {
    rc |= cznn::make_map_2d(&t->map_wf[l], t->wf16[l], C, 9LL * C, cznn::conv_tile_n(C, false));
    rc |= cznn::make_map_2d(&t->map_wd[l], t->wd16[l], C, 9LL * C, cznn::conv_tile_n(C, false));
  }
  if (rc) { delete h; return CZ_ERR_CUDA; }
  k_fill<<<blocks_for(t->maxb), 256, 0, t->st>>>(t->ones, t->maxb, 1.f);
  if (cudaGetLastError() != cudaSuccess) { delete h; return cz_fail(CZ_ERR_CUDA, "cz_train_create: launch failed"); }
  *out = h;
  return 0;
}

void cz_train_destroy(cz_trainer* h) { delete h; }

static const cz_tensor_desc* find_desc(const cz_tensor_desc* d, int n, const Param& q) {
  return cznn::find_keras_tensor(d, n, q.layer, q.weight);
}

int cz_train_set_params(cz_trainer* h, const cz_tensor_desc* params, int32_t n, const cz_tensor_desc* velocity, int32_t nv) {
  if (!h) return cz_fail(CZ_ERR_ARG, "cz_train_set_params: null trainer");
  if (!params || n <= 0 || !velocity || nv <= 0) return cz_fail(CZ_ERR_ARG, "cz_train_set_params: empty tensor list");
  Trainer* t = &h->t;
  std::vector<float*> w(t->p.size()), v(t->p.size());
  for (size_t i = 0; i < t->p.size(); ++i) {
    const Param& q = t->p[i];
    const cz_tensor_desc* d = find_desc(params, n, q);
    if (!d || !d->dev || d->numel != q.numel)
      return cz_fail(CZ_ERR_ARG, "cz_train_set_params: missing or mis-sized tensor %s/%s (want %lld)", q.layer.c_str(), q.weight.c_str(), q.numel);
    w[i] = (float*)d->dev;
    if (q.train) {
      const cz_tensor_desc* dv = find_desc(velocity, nv, q);
      if (!dv || !dv->dev || dv->numel != q.numel)
        return cz_fail(CZ_ERR_ARG, "cz_train_set_params: missing or mis-sized velocity %s/%s (want %lld)", q.layer.c_str(), q.weight.c_str(), q.numel);
      v[i] = (float*)dv->dev;
    }
  }
  for (size_t i = 0; i < t->p.size(); ++i) { t->p[i].w = w[i]; t->p[i].v = v[i]; }
  t->params_set = true;
  t->adam = false;                   // the Adam table points at the previous weights: register it again
  return 0;
}

int cz_train_step(cz_trainer* h, const float* planes, const float* policy_target, const float* value_target, int32_t batch,
                  const cz_train_hparams* hp, float* losses) {
  if (!h) return cz_fail(CZ_ERR_ARG, "cz_train_step: null trainer");
  Trainer* t = &h->t;
  if (!t->params_set) return cz_fail(CZ_ERR_STATE, "cz_train_step: parameters not set (cz_train_set_params)");
  if (batch < 1 || batch > t->maxb) return cz_fail(CZ_ERR_ARG, "cz_train_step: batch %d outside 1..%d", batch, t->maxb);
  if (!planes || !policy_target || !value_target || !hp || !losses) return cz_fail(CZ_ERR_ARG, "cz_train_step: null pointer");
  if (hp->struct_bytes != (int)sizeof(cz_train_hparams)) return cz_fail(CZ_ERR_ARG, "cz_train_step: hparams struct_bytes mismatch");
  const int rc = step(t, planes, policy_target, value_target, batch, *hp, losses);
  if (!rc && t->adam) ++t->iterations;
  return rc;
}

int cz_train_set_adam(cz_trainer* h, const cz_tensor_desc* m, int32_t nm, const cz_tensor_desc* v, int32_t nv, double beta_1,
                      double beta_2, double epsilon) {
  if (!h) return cz_fail(CZ_ERR_ARG, "cz_train_set_adam: null trainer");
  Trainer* t = &h->t;
  if (!t->params_set) return cz_fail(CZ_ERR_STATE, "cz_train_set_adam: parameters not set (cz_train_set_params)");
  if (!m || nm <= 0 || !v || nv <= 0) return cz_fail(CZ_ERR_ARG, "cz_train_set_adam: empty tensor list");
  if (!(beta_1 >= 0.0 && beta_1 < 1.0) || !(beta_2 >= 0.0 && beta_2 < 1.0) || !(epsilon >= 0.0))
    return cz_fail(CZ_ERR_ARG, "cz_train_set_adam: beta_1, beta_2 must lie in [0, 1) and epsilon >= 0");
  std::vector<AdamSeg> segs;
  std::vector<float*> am(t->p.size(), nullptr), av(t->p.size(), nullptr);
  long long blocks = 0;
  for (size_t i = 0; i < t->p.size(); ++i) {
    const Param& q = t->p[i];
    if (!q.train) continue;
    const cz_tensor_desc* dm = find_desc(m, nm, q);
    const cz_tensor_desc* dv = find_desc(v, nv, q);
    if (!dm || !dm->dev || dm->numel != q.numel || !dv || !dv->dev || dv->numel != q.numel)
      return cz_fail(CZ_ERR_ARG, "cz_train_set_adam: missing or mis-sized moment %s/%s (want %lld)", q.layer.c_str(), q.weight.c_str(), q.numel);
    am[i] = (float*)dm->dev; av[i] = (float*)dv->dev;
    segs.push_back(AdamSeg{q.w, am[i], av[i], q.g, q.numel, blocks, q.reg ? 1 : 0, 0});
    blocks += (q.numel + kAdamChunk - 1) / kAdamChunk;
  }
  if (blocks > 0x7fffffffLL) return cz_fail(CZ_ERR_UNSUPPORTED, "cz_train_set_adam: %lld update blocks", blocks);
  t->adam_host = segs;
  CZ_CUDA(cudaMemcpyAsync(t->adam_tab, t->adam_host.data(), segs.size() * sizeof(AdamSeg), cudaMemcpyHostToDevice, t->st));
  CZ_CUDA(cudaStreamSynchronize(t->st));
  for (size_t i = 0; i < t->p.size(); ++i) { t->p[i].am = am[i]; t->p[i].av = av[i]; }
  t->n_adam = (int)segs.size(); t->adam_blocks = blocks;
  t->b1 = beta_1; t->b2 = beta_2; t->eps = epsilon;
  t->iterations = 0;
  t->adam = true;
  return 0;
}

int cz_train_adam_iterations(cz_trainer* h, int64_t* out) {
  if (!h || !out) return cz_fail(CZ_ERR_ARG, "cz_train_adam_iterations: null argument");
  if (!h->t.adam) return cz_fail(CZ_ERR_STATE, "cz_train_adam_iterations: the trainer does not use Adam");
  *out = h->t.iterations;
  return 0;
}

int cz_train_read_grad(cz_trainer* h, const char* name, void* dst, int64_t numel) {
  if (!h || !name || !dst) return cz_fail(CZ_ERR_ARG, "cz_train_read_grad: null argument");
  Trainer* t = &h->t;
  const cz_tensor_desc named = {name, nullptr, 0};
  for (const Param& q : t->p) {
    if (!q.train || !find_desc(&named, 1, q)) continue;
    if (numel != q.numel) return cz_fail(CZ_ERR_ARG, "cz_train_read_grad: %s has %lld elements, not %lld", name, q.numel, (long long)numel);
    CZ_CUDA(cudaMemcpyAsync(dst, q.g, (size_t)numel * 4, cudaMemcpyDeviceToDevice, t->st));
    CZ_CUDA(cudaStreamSynchronize(t->st));
    return 0;
  }
  return cz_fail(CZ_ERR_ARG, "cz_train_read_grad: no trainable tensor named %s", name);
}

// Tests: copy an intermediate buffer as the last step left it (cz_train_buffer in the header lists what each holds).
int cz_train_read_buffer(cz_trainer* h, int32_t which, int32_t index, void* dst, int64_t dst_bytes, int64_t* bytes) {
  if (!h) return cz_fail(CZ_ERR_ARG, "cz_train_read_buffer: null trainer");
  Trainer* t = &h->t;
  if (t->last_batch < 1) return cz_fail(CZ_ERR_STATE, "cz_train_read_buffer: no step has run");
  const long long n = t->last_batch, P = n * 90, C = t->C, L = t->L;
  const long long nbn = (long long)t->bn.size();
  long long lim = 1;                              // valid indices are 0 .. lim - 1
  switch (which) {
    case CZ_TRAIN_BUF_BLOCK_OUT32: case CZ_TRAIN_BUF_BLOCK_OUT16: lim = L + 1; break;
    case CZ_TRAIN_BUF_CONV1_OUT16: lim = L; break;
    case CZ_TRAIN_BUF_BN_MEAN: case CZ_TRAIN_BUF_BN_VAR: case CZ_TRAIN_BUF_BN_DZ: lim = nbn; break;
    default: break;
  }
  if (index < 0 || index >= lim) return cz_fail(CZ_ERR_ARG, "cz_train_read_buffer: index %d of buffer %d outside 0..%lld", index, which, lim - 1);
  const void* src = nullptr;
  long long nb = 0;
  switch (which) {
    case CZ_TRAIN_BUF_PLANE_INDEX: src = t->pl; nb = n * 2 * 90; break;
    case CZ_TRAIN_BUF_BLOCK_OUT32: src = t->s32[index]; nb = P * C * 4; break;
    case CZ_TRAIN_BUF_BLOCK_OUT16: src = t->a16[index]; nb = P * C * 2; break;
    case CZ_TRAIN_BUF_CONV1_OUT16: src = t->h16[index]; nb = P * C * 2; break;
    case CZ_TRAIN_BUF_BN_MEAN: src = t->bn[index].mean; nb = t->bn[index].C * 4LL; break;
    case CZ_TRAIN_BUF_BN_VAR: src = t->bn[index].var; nb = t->bn[index].C * 4LL; break;
    case CZ_TRAIN_BUF_BN_DZ: src = t->bn[index].z; nb = P * t->bn[index].C * 4; break;
    case CZ_TRAIN_BUF_POL_FEAT: src = t->Fp; nb = n * t->pc * 90 * 4; break;
    case CZ_TRAIN_BUF_VAL_FEAT: src = t->Fv; nb = n * t->vc * 90 * 4; break;
    case CZ_TRAIN_BUF_LOGITS: src = t->logits; nb = n * kLabels * 4; break;
    case CZ_TRAIN_BUF_DLOGITS: src = t->dlog; nb = n * kLabels * 4; break;
    case CZ_TRAIN_BUF_VAL_HIDDEN_PRE: src = t->hpre; nb = n * t->H * 4; break;
    case CZ_TRAIN_BUF_VAL_HIDDEN: src = t->hact; nb = n * t->H * 4; break;
    case CZ_TRAIN_BUF_DVAL_HIDDEN: src = t->dh; nb = n * t->H * 4; break;
    case CZ_TRAIN_BUF_VAL_PRE: src = t->vpre; nb = n * 4; break;
    case CZ_TRAIN_BUF_DVAL_PRE: src = t->dvpre; nb = n * 4; break;
    case CZ_TRAIN_BUF_CE_ROWS: src = t->ce_rows; nb = n * 4; break;
    case CZ_TRAIN_BUF_SE_ROWS: src = t->se_rows; nb = n * 4; break;
    case CZ_TRAIN_BUF_DPOL_FEAT: src = t->dF; nb = n * t->pc * 90 * 4; break;
    case CZ_TRAIN_BUF_TRUNK_GRAD: src = t->G; nb = P * C * 4; break;
    case CZ_TRAIN_BUF_SCALE_SLOTS: src = t->scale_slots; nb = (2 * L + 1) * 4 * 4; break;
    default: return cz_fail(CZ_ERR_ARG, "cz_train_read_buffer: unknown buffer %d", which);
  }
  if (bytes) *bytes = nb;
  if (!dst) return 0;
  if (dst_bytes < nb) return cz_fail(CZ_ERR_ARG, "cz_train_read_buffer: %lld bytes < %lld", (long long)dst_bytes, nb);
  CZ_CUDA(cudaMemcpyAsync(dst, src, (size_t)nb, cudaMemcpyDeviceToDevice, t->st));
  CZ_CUDA(cudaStreamSynchronize(t->st));
  return 0;
}

// ---- stage building blocks (tests): each runs the step's own launch sequence for one stage on caller buffers.
// 3x3 conv gradients on dense activations [n][90][c]: dy f32, x fp16; dw out Keras HWIO f32 [3][3][c][c]
int cz_train_wgrad3x3(const void* x16, const float* dy, int n, int c, float* dw, void* stream) {
  if (c % 64 || c < 64 || c > 256 || n < 1) return cz_fail(CZ_ERR_ARG, "cz_train_wgrad3x3: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  const long long P = (long long)n * 90;
  __half* d16 = nullptr; float *part = nullptr, *slot = nullptr;
  CZ_CUDA(cudaMalloc(&d16, P * c * 2));
  CZ_CUDA(cudaMalloc(&part, (size_t)kMaxSplits * 9 * c * c * 4));
  CZ_CUDA(cudaMalloc(&slot, 16));
  CUtensorMap mdy, mx;
  int rc = cznn::make_map_2d(&mdy, d16, c, P, wgrad::kPix);
  if (!rc) rc = cznn::make_map_im2col(&mx, x16, c, n, wgrad::kPix);
  if (!rc) {
    cudaMemsetAsync(slot, 0, 16, st);
    k_absmax<<<blocks_for(P * c), 256, 0, st>>>(dy, P * c, reinterpret_cast<unsigned*>(slot));
    k_pick_scale<<<1, 1, 0, st>>>(slot);
    k_to_half_scaled<<<blocks_for(P * c), 256, 0, st>>>(dy, P * c, slot, d16);
    rc = wgrad_launch(c, n, mdy, mx, part, slot, dw, st);
  }
  cudaStreamSynchronize(st);
  cudaFree(d16); cudaFree(part); cudaFree(slot);
  return rc;
}
// dx f32 [n][90][c] = conv^T(dy, W) for W Keras HWIO f32
int cz_train_dgrad3x3(const float* dy, const float* w_hwio, int n, int c, float* dx, void* stream) {
  if (c % 64 || c < 64 || c > 256 || n < 1) return cz_fail(CZ_ERR_ARG, "cz_train_dgrad3x3: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  const long long P = (long long)n * 90;
  __half *d16 = nullptr, *wf = nullptr, *wd = nullptr; float* slot = nullptr;
  CZ_CUDA(cudaMalloc(&d16, P * c * 2));
  CZ_CUDA(cudaMalloc(&wf, 9ULL * c * c * 2));
  CZ_CUDA(cudaMalloc(&wd, 9ULL * c * c * 2));
  CZ_CUDA(cudaMalloc(&slot, 16));
  CUtensorMap ma, mb;
  int rc = cznn::make_map_2d(&ma, d16, c, P, igemm::kHaloBox);
  if (!rc) rc = cznn::make_map_2d(&mb, wd, c, 9LL * c, cznn::conv_tile_n(c, false));
  if (!rc) {
    cudaMemsetAsync(slot, 0, 16, st);
    k_prep_conv3_train<<<blocks_for(9LL * c * c), 256, 0, st>>>(w_hwio, wf, wd, c);
    k_absmax<<<blocks_for(P * c), 256, 0, st>>>(dy, P * c, reinterpret_cast<unsigned*>(slot));
    k_pick_scale<<<1, 1, 0, st>>>(slot);
    k_to_half_scaled<<<blocks_for(P * c), 256, 0, st>>>(dy, P * c, slot, d16);
    rc = conv3x3(n, c, ma, mb, dx, st);
    if (!rc) k_scale<<<blocks_for(P * c), 256, 0, st>>>(dx, P * c, slot + 2);
  }
  cudaStreamSynchronize(st);
  cudaFree(d16); cudaFree(wf); cudaFree(wd); cudaFree(slot);
  if (!rc && cudaGetLastError() != cudaSuccess) rc = cz_fail(CZ_ERR_CUDA, "cz_train_dgrad3x3: launch failed");
  return rc;
}
// BatchNormalization (training mode) + optional fp32 skip + ReLU on z [rows][c]: out f32, batch mean / biased var [c].
// With `up` (gradient of the ReLU output) also the backward: dz [rows][c], dgamma, dbeta [c].
int cz_train_bn(const float* z, long long rows, int c, const float* gamma, const float* beta, const float* skip, float* out,
                float* mean, float* var, const float* up, float* dz, float* dgamma, float* dbeta, void* stream) {
  if (rows < 1 || c < 1 || c > 256 || !z || !gamma || !beta || !mean || !var) return cz_fail(CZ_ERR_ARG, "cz_train_bn: bad arguments");
  if (up && (!dz || !dgamma || !dbeta)) return cz_fail(CZ_ERR_ARG, "cz_train_bn: backward needs dz, dgamma and dbeta");
  Trainer t;
  t.st = (cudaStream_t)stream;
  float *part = nullptr, *rstd = nullptr;
  CZ_CUDA(cudaMalloc(&part, (size_t)1024 * 2 * 256 * 4));
  CZ_CUDA(cudaMalloc(&rstd, (size_t)c * 4));
  t.col_part = part;
  t.p.push_back(Param{"", "gamma", c, true, false, const_cast<float*>(gamma), nullptr, dgamma});
  t.p.push_back(Param{"", "beta", c, true, false, const_cast<float*>(beta), nullptr, dbeta});
  Bn b; memset(&b, 0, sizeof(b));
  b.C = c; b.gamma = 0; b.beta = 1; b.z = const_cast<float*>(z); b.mean = mean; b.var = var; b.rstd = rstd;
  int rc = bn_forward(&t, b, rows, skip, nullptr, out, 0);
  if (!rc && up) {
    CZ_CUDA(cudaMemcpyAsync(dz, z, (size_t)rows * c * 4, cudaMemcpyDeviceToDevice, t.st));
    b.z = dz;                                       // the backward writes dz over its input
    rc = bn_backward(&t, b, rows, skip, up, nullptr, 0, nullptr, nullptr);
  }
  cudaStreamSynchronize(t.st);
  cudaFree(part); cudaFree(rstd);
  return rc;
}

}  // extern "C"
