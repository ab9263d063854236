// cz_igemm.cuh — the one dense contraction of the hot path: implicit-GEMM 3x3 convolution (and the
// plain GEMM of the policy head) on Hopper warpgroup tensor cores (wgmma), TMA-fed operands.
//
// Replaces the Conv2D/BatchNormalization/Add/Activation stack of agent/model.py:68-83 (residual
// block) and the Dense of :54 (policy_out) that the reference runs through Keras/TF/cuDNN.
//
// Operand A in HBM (fp16):
//   conv (conv == 1): activations [n_boards*90][C] pixels, channels contiguous.  A 3x3 tap (dy,dx) of 128 consecutive output
//          pixels is ONE im2col-mode TMA load (64 channels x 128 pixels); taps outside the board are zero-filled by the TMA
//          unit and the 128-pixel column walks across rows and boards.
//   GEMM   (conv == 0): A [M][K] rows, 128 per tile.
// Tile: M = 128 pixels / rows, N = N_TILE output channels (<= 256), K walks taps x C_in in 64-channel blocks (128-byte
//   swizzled rows).  Every output element accumulates its K blocks in the same order whatever the tile shape, so results do
//   not depend on N_TILE or on how the M tiles are spread over CTAs.
// CTA = 3 warpgroups: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers, each issuing m64nN wgmma
//   on its 64 rows of the tile with fp32 accumulators in registers, then running the epilogue from those registers
//   (+bias (+residual) -> ReLU -> fp16 / fp32 -> HBM).  kStages-deep smem ring with full/empty mbarriers; the producer runs
//   ahead into the next tile while the consumers store the current one.  Persistent: grid <= #SMs, tiles strided over CTAs.
//   After the role split the producer warpgroup gives its registers to the consumers (setmaxnreg).
// Staged epilogue (Args::staged: conv without a skip stream, fp16 out, M tiles that lie wholly inside the batch): the
//   tile leaves in 32-column steps through a small ring of slots per consumer warpgroup.  A slot holds 64 rows x 32 fp16
//   columns (64-byte rows, SWIZZLE_64B, as the output's tensor map expects); the warpgroup writes a step into a slot and one
//   thread hands it to a TMA store, so the stores are whole sectors and drain while the next tile's MMAs run.  The arithmetic
//   per element is that of the register epilogue, which everything else keeps: the convs with a skip stream (loading it by
//   TMA into the ring was measured and did not pay, DESIGN.md 3.1), and the last, partial M tile, because a tensor store
//   clips at the buffer's extent, not at the device-side batch.
#pragma once
#include <cuda_fp16.h>
#include "cz_wgmma.cuh"

namespace igemm {

constexpr int kBlockK = 64;                 // fp16 per k-block row = 128 B = swizzle span
constexpr int kTileM = 128;
constexpr int kAStageBytes = kTileM * 128;  // 16 KB
constexpr int kThreads = 384;
constexpr int kConsumerWarps = 8;
constexpr int kSmemLimit = 232448;          // opt-in dynamic shared memory per CTA on sm_90 (227 KB)
constexpr int kMaxStages = 8;
constexpr int kEpiCols = 32;                       // columns per step of the staged epilogue
constexpr int kEpiSlotBytes = 64 * kEpiCols * 2;   // 4 KB: 64 rows x 32 fp16
constexpr int kEpiSlots = 3;                       // per consumer warpgroup: one being written, two being stored
constexpr int kEpiBytes = kEpiSlots * kEpiSlotBytes;

struct Args {
  int n_taps;        // 9 (3x3 conv) or 1 (plain GEMM)
  int k_chunks;      // C_in / 64
  int m_tiles;       // ceil(rows / kTileM): the host's grid bound (an upper bound when n_dev is set)
  int n_tiles;       // ceil(N / N_TILE)
  int rows;          // conv: pixels (n_boards*90); GEMM: M
  int n_total;       // B-operand rows per tap (C_out padded to N_TILE multiple)
  int n_valid;       // real number of output columns
  int ldo;           // output leading dimension in elements
  int conv;          // 1: 3x3 conv over [B*90][C] pixels fed by im2col TMA; 0: GEMM
  int relu;
  int out_f32;       // 1: float output (GEMM logits), 0: fp16
  const float* bias; // [n_total] or null
  const __half* residual;  // same layout as out (fp16) or null
  const float* residual32; // fp32 skip stream (takes precedence over `residual`) or null
  float* out32;            // optional fp32 copy of the output (the skip stream of the next block) or null
  void* out;
  // Batch size read on the DEVICE (fixed-shape launches: the host never learns how many leaves a wave produced).  When
  // n_dev != null, rows = *n_dev * rows_per_unit and m_tiles follows; `rows` / `m_tiles` above are then only upper bounds.
  const int* n_dev;
  int rows_per_unit; // 90 pixels per board (conv), 1 (GEMM rows = positions)
  // GEMM mode (out_f32): per output row and N tile the pair {max_j x_j, sum_j exp(x_j - max)} over the tile's valid
  // columns — the softmax is finished by whoever reads the logits (k_softmax / k_legal_priors), never a second full pass
  float2* row_stats; // [rows][n_tiles] or null
  int staged;        // conv, fp16 out, no skip: tmOut is valid, full M tiles take the staged epilogue
};

// rows / m-tiles of this launch (device-side batch size)
__device__ __forceinline__ int args_rows(const Args& a) { return a.n_dev ? __ldg(a.n_dev) * a.rows_per_unit : a.rows; }

// Shared memory: the epilogue ring of both consumer warpgroups, then as many operand stages as still fit
template <int N_TILE>
struct Cfg {
  static constexpr int kBStageBytes = N_TILE * 128;
  static constexpr int kStageBytes = kAStageBytes + kBStageBytes;
  static constexpr int kFit = (kSmemLimit - 2 * kEpiBytes - 256 - 1024) / kStageBytes;
  static constexpr int kStages = kFit > kMaxStages ? kMaxStages : kFit;   // 4 (N = 256) .. 8 (N = 64)
  static constexpr int kSmemBytes = kStages * kStageBytes + 2 * kEpiBytes + 256 + 1024;    // + barriers + alignment slack
  static_assert(N_TILE % 64 == 0 && N_TILE <= 256, "wgmma N tile");
  static_assert((2 * kStages + 2 * kEpiSlots) * 8 <= 256, "barrier space");
};

template <int N_TILE>
__global__ void __launch_bounds__(kThreads, 1)
k_igemm(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
        const Args a) {
  using C = Cfg<N_TILE>;
  constexpr int S = C::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* epi = smem + S * C::kStageBytes;                                   // [2 warpgroups][kEpiBytes]
  uint64_t* full = reinterpret_cast<uint64_t*>(epi + 2 * kEpiBytes);          // [S]  TMA -> MMA
  uint64_t* empty = full + S;                                                 // [S]  MMA -> TMA (one arrive per consumer warp)
  uint64_t* efree = empty + S;    // [2][kEpiSlots]  the slot's last store has read it: the warpgroup may write it again

  const int wgi = threadIdx.x >> 7, t = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { wg::mbar_init(&full[s], 1); wg::mbar_init(&empty[s], kConsumerWarps); }
    for (int s = 0; s < 2 * kEpiSlots; ++s) wg::mbar_init(&efree[s], 1);
    wg::fence_barrier_init();
  }
  wg::griddep_launch_dependents();     // (PDL launches only) the next conv may become resident while this one runs
  __syncthreads();
  wg::griddep_wait();                  // (PDL launches only) the producer of this conv's input has completed

  const int n_kb = a.n_taps * a.k_chunks;
  const int rows = args_rows(a);
  const int m_tiles = (rows + kTileM - 1) / kTileM;
  const int total_tiles = m_tiles * a.n_tiles;

  constexpr int kSteps = N_TILE / kEpiCols;                // steps of the staged epilogue per tile
  auto tile_staged = [&](int tile) { return a.staged && (tile % m_tiles) * kTileM + kTileM <= rows; };

  if (wgi == 0) {
    // ------------------------------------------------------------ TMA producer
    wg::reg_dealloc<40>();
    if (t == 0) {
      wg::prefetch_tmap(&tmA);
      wg::prefetch_tmap(&tmB);
      // Conv with a skip stream: the epilogue reads the tile's skip rows right after the last MMA, when every CTA of the
      // wave does the same, so the reads would all miss L2 at once with the tensor cores idle.  Halfway through the tile's
      // main loop the producer prefetches them into L2 instead (rows below args_rows only; at N_TILE = ldo one contiguous
      // range, else one range per row).  Halfway rather than at the tile's first load: the first load is issued while the
      // previous tile's epilogue still has to stream its outputs through L2, which could evict the prefetched lines.
      const uint8_t* skip = !a.conv ? nullptr : a.residual32 ? reinterpret_cast<const uint8_t*>(a.residual32)
                                                               : reinterpret_cast<const uint8_t*>(a.residual);
      const int skip_es = a.residual32 ? 4 : 2;
      uint32_t s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m_tile = tile % m_tiles, n_tile = tile / m_tiles;
        // conv: first output pixel of this tile as (image, row, column); im2col walks on from there
        const int pix0 = m_tile * kTileM, img0 = pix0 / 90, row0 = (pix0 % 90) / 9, col0 = pix0 % 9;
        for (int tap = 0; tap < a.n_taps; ++tap) {
          const int dy = a.n_taps == 9 ? tap / 3 - 1 : 0;
          const int dx = a.n_taps == 9 ? tap % 3 - 1 : 0;
          for (int kc = 0; kc < a.k_chunks; ++kc) {
            if (skip && tap * a.k_chunks + kc == n_kb / 2) {
              const int nr = min(kTileM, rows - pix0);
              const uint8_t* p0 = skip + ((long long)pix0 * a.ldo + n_tile * N_TILE) * skip_es;
              if (N_TILE == a.ldo)
                wg::prefetch_l2_bulk(p0, (uint32_t)(nr * N_TILE * skip_es));
              else
                for (int r = 0; r < nr; ++r) wg::prefetch_l2_bulk(p0 + (long long)r * a.ldo * skip_es, N_TILE * skip_es);
            }
            wg::mbar_wait(&empty[s], ph ^ 1);
            uint8_t* sA = smem + s * C::kStageBytes;
            uint8_t* sB = sA + kAStageBytes;
            wg::mbar_expect_tx(&full[s], (uint32_t)C::kStageBytes);
            if (a.conv)
              wg::tma_load_im2col_4d(sA, &tmA, &full[s], kc * kBlockK, col0 - 1, row0 - 1, img0, (uint16_t)(dx + 1), (uint16_t)(dy + 1));
            else
              wg::tma_load_2d(sA, &tmA, &full[s], kc * kBlockK, m_tile * kTileM);
            wg::tma_load_2d(sB, &tmB, &full[s], kc * kBlockK, tap * a.n_total + n_tile * N_TILE);
            if (++s == (uint32_t)S) { s = 0; ph ^= 1; }
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers: MMA + epilogue on rows cw*64 .. cw*64+63
  wg::reg_alloc<232>();
  const int cw = wgi - 1, warp = t >> 5, lane = t & 31;
  const int mrow = cw * 64 + warp * 16 + (lane >> 2);       // accumulator rows mrow and mrow + 8 of the tile
  const int cq = 2 * (lane & 3);                            // first of the two adjacent columns per 8-column group
  float acc[N_TILE / 2];
  // staged epilogue: this warpgroup's slots and barriers; byte offset of this thread's first row (warp * 16 + lane / 4 of the
  // warpgroup's 64; the second is 8 rows on, same swizzle phase) and column pair inside a slot, before the swizzle XOR
  uint8_t* ering = epi + cw * kEpiBytes;
  uint64_t* fre = efree + cw * kEpiSlots;
  const uint32_t erow = warp * 16 + (lane >> 2);
  const uint32_t e_off = erow * 64 + (lane & 3) * 4, e_x = (erow >> 1) & 3;
  uint32_t e_slot = 0, e_ph = 0;                              // the next step's slot and its parity
  uint32_t e_issued = 0, e_released = 0, e_rel_slot = 0;      // (thread 0 of the warpgroup) steps stored / slots handed back
  auto release_to = [&](uint32_t upto) {                      // the stores of steps < upto have read their slots
    for (; e_released < upto; ++e_released) {
      wg::mbar_arrive(&fre[e_rel_slot]);
      if (++e_rel_slot == kEpiSlots) e_rel_slot = 0;
    }
  };
  uint32_t s = 0, ph = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int m_tile = tile % m_tiles, n_tile = tile / m_tiles;
    uint32_t prev = 0;
    for (int kb = 0; kb < n_kb; ++kb) {
      wg::mbar_wait(&full[s], ph);
      const uint32_t sA = wg::smem_u32(smem + s * C::kStageBytes);
      const uint64_t da = wg::smem_desc_sw128(sA + cw * 64 * 128);
      const uint64_t db = wg::smem_desc_sw128(sA + kAStageBytes);
      wg::wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)                // +32 B per k16 step inside the swizzle atom
        wg::Wgmma<N_TILE>::mma(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb | k) != 0);
      wg::wgmma_commit();
      wg::wgmma_wait<1>();                                  // the previous stage's MMAs are done: hand it back to the producer
      if (kb > 0 && lane == 0) wg::mbar_arrive(&empty[prev]);
      prev = s;
      if (++s == (uint32_t)S) { s = 0; ph ^= 1; }
    }
    wg::wgmma_wait<0>();
    if (lane == 0) wg::mbar_arrive(&empty[prev]);

    // ------------------------------------------------------------ epilogue
    const int nb = n_tile * N_TILE + cq;                    // column of acc[4j + 2h] is nb + 8j
    if (a.bias) {
#pragma unroll
      for (int j = 0; j < N_TILE / 8; ++j) {                // bias arrays are padded to the N tile
        const float2 b = __ldg(reinterpret_cast<const float2*>(a.bias + nb + 8 * j));
        acc[4 * j] += b.x; acc[4 * j + 1] += b.y; acc[4 * j + 2] += b.x; acc[4 * j + 3] += b.y;
      }
    }
    if (tile_staged(tile)) {
      if (t == 0) { wg::bulk_wait_group_read<0>(); release_to(e_issued); }    // the previous tile's last slots
#pragma unroll
      for (int st = 0; st < kSteps; ++st) {
        uint8_t* slot = ering + e_slot * kEpiSlotBytes;
        wg::mbar_wait(&fre[e_slot], e_ph ^ 1);              // passes on a slot that has not been used yet
#pragma unroll
        for (int jj = 0; jj < kEpiCols / 8; ++jj) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int i = 4 * (st * (kEpiCols / 8) + jj) + 2 * h;
            float x0 = acc[i], x1 = acc[i + 1];
            if (a.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
            *reinterpret_cast<__half2*>(slot + e_off + h * 8 * 64 + ((jj ^ e_x) << 4)) = __floats2half2_rn(x0, x1);
          }
        }
        wg::fence_proxy_async();
        wg::named_barrier(1 + cw, 128);
        if (t == 0) {
          wg::tma_store_2d(&tmOut, slot, n_tile * N_TILE + st * kEpiCols, m_tile * kTileM + cw * 64);
          wg::bulk_commit();
          ++e_issued;
          // hand back the previous step's slot (its store has had this step's time to read it); this step's store stays in flight
          wg::bulk_wait_group_read<1>();
          release_to(e_issued - 1);
        }
        if (++e_slot == kEpiSlots) { e_slot = 0; e_ph ^= 1; }
      }
      continue;
    }
    // accumulator row mrow + 8h: global output row (pixel / GEMM row), and whether it is inside the batch
    auto out_row = [&](int h, long long& grow, bool& valid) {
      grow = (long long)m_tile * kTileM + mrow + 8 * h;
      valid = grow < rows;
    };
    // + skip stream, for both rows before the first output store.  The compiler keeps every load behind the stores that
    // precede it (a store might alias the skip stream), so loads interleaved with the stores would go out one round trip
    // at a time; here they go out back to back.  Same operations in the same order: (acc + bias) + skip.
    if (!a.out_f32 && (a.residual32 || a.residual)) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        long long grow;
        bool valid;
        out_row(h, grow, valid);
        if (!valid) continue;
        if (a.residual32) {
          const float* r32 = a.residual32 + grow * a.ldo;
#pragma unroll
          for (int j = 0; j < N_TILE / 8; ++j) {
            const float2 r = __ldg(reinterpret_cast<const float2*>(r32 + nb + 8 * j));
            acc[4 * j + 2 * h] += r.x; acc[4 * j + 2 * h + 1] += r.y;
          }
        } else {
          const __half* r16 = a.residual + grow * a.ldo;
#pragma unroll
          for (int j = 0; j < N_TILE / 8; ++j) {
            const float2 r = __half22float2(__ldg(reinterpret_cast<const __half2*>(r16 + nb + 8 * j)));
            acc[4 * j + 2 * h] += r.x; acc[4 * j + 2 * h + 1] += r.y;
          }
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      long long grow;                                       // global output row
      bool valid;
      out_row(h, grow, valid);
      if (a.out_f32) {
        if (a.row_stats) {                                  // the 4 threads of a quad hold one row: reduce across them
          float mx = -INFINITY;
#pragma unroll
          for (int j = 0; j < N_TILE / 8; ++j) {
            if (nb + 8 * j < a.n_valid) mx = fmaxf(mx, acc[4 * j + 2 * h]);
            if (nb + 8 * j + 1 < a.n_valid) mx = fmaxf(mx, acc[4 * j + 2 * h + 1]);
          }
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          float sum = 0.f;
#pragma unroll
          for (int j = 0; j < N_TILE / 8; ++j) {
            if (nb + 8 * j < a.n_valid) sum += __expf(acc[4 * j + 2 * h] - mx);
            if (nb + 8 * j + 1 < a.n_valid) sum += __expf(acc[4 * j + 2 * h + 1] - mx);
          }
          sum += __shfl_xor_sync(0xffffffffu, sum, 1);
          sum += __shfl_xor_sync(0xffffffffu, sum, 2);
          if (valid && (lane & 3) == 0) a.row_stats[grow * a.n_tiles + n_tile] = make_float2(mx, sum);
        }
        if (!valid) continue;
        float* o = reinterpret_cast<float*>(a.out) + grow * a.ldo;
#pragma unroll
        for (int j = 0; j < N_TILE / 8; ++j) {
          const int n = nb + 8 * j;
          float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
          if (a.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
          if (n + 1 < a.n_valid) *reinterpret_cast<float2*>(o + n) = make_float2(x0, x1);
          else if (n < a.n_valid) o[n] = x0;
        }
      } else {
        if (!valid) continue;
        __half* o = reinterpret_cast<__half*>(a.out) + grow * a.ldo;
        float* o32 = a.out32 ? a.out32 + grow * a.ldo : nullptr;
#pragma unroll
        for (int j = 0; j < N_TILE / 8; ++j) {
          const int n = nb + 8 * j;
          float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
          if (a.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
          *reinterpret_cast<__half2*>(o + n) = __floats2half2_rn(x0, x1);
          if (o32) *reinterpret_cast<float2*>(o32 + n) = make_float2(x0, x1);
        }
      }
    }
  }
  if (t == 0) wg::bulk_wait_group_all();                    // the staged stores have landed before the grid can count as complete
}

}  // namespace igemm
