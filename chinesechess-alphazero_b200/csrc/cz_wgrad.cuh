// cz_wgrad.cuh — weight gradient of a 3x3 "same" convolution on Hopper warpgroup tensor cores:
//
//   dW[tap][co][ci] = sum_p dy[p][co] * x[p + tap][ci]        (p = pixel of the batch, B*90 of them)
//
// a GEMM with M = co, N = ci and K = pixels.  Both operands arrive by TMA with channels contiguous, which makes them
// MN-major in shared memory (wgmma tnspA = tnspB = 1):
//   dy  fp16 [P][C], tiled 2D box {64 co, 64 pixels}
//   x   fp16 [n][10][9][C], the forward's im2col-mode load with a 64-pixel box: row r of the box is x at pixel p0 + r moved
//       by the tap, off-board taps zero-filled by the TMA unit; pixels past the batch read as zeros on both sides.
// Work item = (tap, 128-row co tile, K split).  One CTA per item: warpgroup 0 = TMA producer, warpgroups 1 and 2 take the
// two 64-row halves of the co tile (the second idles when the tile has only 64 rows) and hold all C columns as NB = C/64
// m64n64 accumulators.  Each split writes fp32 partials part[split][tap][co][ci]; k_wgrad_reduce (cz_train.cu) sums the
// splits in a fixed order, so a step is bit-reproducible.
#pragma once
#include <cuda_fp16.h>
#include "cz_wgmma.cuh"

namespace wgrad {

constexpr int kPix = 64;                        // pixels (K) per stage
constexpr int kBox = kPix * 128;                // one {64 channels x 64 pixels} fp16 box: 8 KB
constexpr int kThreads = 384;
constexpr int kConsumerWarps = 8;
constexpr int kSmemLimit = 232448;

struct Args {
  int c;             // channels (C_in = C_out)
  int co_tiles;      // ceil(C / 128)
  int chunks;        // ceil(P / 64)
  int splits;        // K splits (<= chunks)
  float* part;       // [splits][9][C][C]
};

template <int NB>
struct Cfg {
  static constexpr int kStageBytes = (2 + NB) * kBox;
  static constexpr int kFit = (kSmemLimit - 256 - 1024) / kStageBytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + 256 + 1024;
};

template <int NB>
__global__ void __launch_bounds__(kThreads, 1)
k_wgrad(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX, const Args a) {
  using Cf = Cfg<NB>;
  constexpr int S = Cf::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * Cf::kStageBytes);
  uint64_t* empty = full + S;

  const int wgi = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int tap = blockIdx.x % 9, co_t = (blockIdx.x / 9) % a.co_tiles, split = blockIdx.x / (9 * a.co_tiles);
  const int co0 = co_t * 128;
  const int n_a = co0 + 64 < a.c ? 2 : 1;      // 64-row halves of the co tile that exist
  const int per = (a.chunks + a.splits - 1) / a.splits;
  const int c0 = split * per, c1 = c0 + per < a.chunks ? c0 + per : a.chunks;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { wg::mbar_init(&full[s], 1); wg::mbar_init(&empty[s], kConsumerWarps); }
    wg::fence_barrier_init();
  }
  __syncthreads();

  if (wgi == 0) {
    if (t == 0) {
      wg::prefetch_tmap(&tmDy);
      wg::prefetch_tmap(&tmX);
      const int kh = tap / 3, kw = tap % 3;
      uint32_t s = 0, ph = 0;
      for (int ch = c0; ch < c1; ++ch) {
        wg::mbar_wait(&empty[s], ph ^ 1);
        uint8_t* base = smem + s * Cf::kStageBytes;
        wg::mbar_expect_tx(&full[s], (uint32_t)((n_a + NB) * kBox));
        const int p0 = ch * kPix, img0 = p0 / 90, row0 = (p0 % 90) / 9, col0 = p0 % 9;
        wg::tma_load_2d(base, &tmDy, &full[s], co0, p0);
        if (n_a > 1) wg::tma_load_2d(base + kBox, &tmDy, &full[s], co0 + 64, p0);
#pragma unroll
        for (int j = 0; j < NB; ++j)
          wg::tma_load_im2col_4d(base + (2 + j) * kBox, &tmX, &full[s], j * 64, col0 - 1, row0 - 1, img0, (uint16_t)kw, (uint16_t)kh);
        if (++s == (uint32_t)S) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  const int cw = wgi - 1, warp = t >> 5, lane = t & 31;
  const bool active = cw < n_a;
  float acc[NB][32];
  uint32_t s = 0, ph = 0, prev = 0;
  for (int ch = c0; ch < c1; ++ch) {
    wg::mbar_wait(&full[s], ph);
    if (active) {
      const uint32_t base = wg::smem_u32(smem + s * Cf::kStageBytes);
      wg::wgmma_fence();
#pragma unroll
      for (int k = 0; k < kPix / 16; ++k) {
        const uint64_t da = wg::smem_desc_sw128_mn(base + cw * kBox + k * 2048);
#pragma unroll
        for (int j = 0; j < NB; ++j)
          wg::WgmmaT<64>::mma(acc[j], da, wg::smem_desc_sw128_mn(base + (2 + j) * kBox + k * 2048), (ch != c0 || k != 0) ? 1u : 0u);
      }
      wg::wgmma_commit();
      wg::wgmma_wait<1>();                      // the previous stage's MMAs are done: hand it back to the producer
      if (ch > c0 && lane == 0) wg::mbar_arrive(&empty[prev]);
    } else if (lane == 0) {
      wg::mbar_arrive(&empty[s]);
    }
    prev = s;
    if (++s == (uint32_t)S) { s = 0; ph ^= 1; }
  }
  if (!active) return;
  wg::wgmma_wait<0>();
  if (c1 <= c0) {
#pragma unroll
    for (int j = 0; j < NB; ++j)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
  }
  // register i of a thread: row warp*16 + lane/4 + 8*((i/2)%2), column 8*(i/4) + 2*(lane%4) + i%2 (Wgmma layout)
  const int row = co0 + cw * 64 + warp * 16 + (lane >> 2);
  float* out = a.part + ((size_t)split * 9 + tap) * a.c * a.c;
#pragma unroll
  for (int j = 0; j < NB; ++j)
#pragma unroll
    for (int q = 0; q < 8; ++q)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int co = row + 8 * h, ci = j * 64 + 8 * q + 2 * (lane & 3);
        *reinterpret_cast<float2*>(out + (size_t)co * a.c + ci) = make_float2(acc[j][4 * q + 2 * h], acc[j][4 * q + 2 * h + 1]);
      }
}

}  // namespace wgrad
