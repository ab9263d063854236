// cz_igemm.cuh — the one dense contraction of the hot path: implicit-GEMM 3x3 convolution (and the
// plain GEMM of the policy head) on Hopper warpgroup tensor cores (wgmma), TMA-fed operands.
//
// Replaces the Conv2D/BatchNormalization/Add/Activation stack of agent/model.py:68-83 (residual
// block) and the Dense of :54 (policy_out) that the reference runs through Keras/TF/cuDNN.
//
// Operand A in HBM (fp16):
//   conv (CONV): activations [n_boards*90][C] pixels, channels contiguous.  An M tile of M_TILE (128 or 256) output pixels
//          starting at pixel pix0 needs the input rows [pix0 - 10, pix0 + M_TILE + 10): a tap (dy, dx) of output pixel p
//          reads input pixel p + 9 dy + dx.  The producer loads those rows ONCE per tile, one chunk per 64 channels (plain
//          2D TMA boxes of kHaloBox rows, 128-byte swizzle; rows before the buffer or past its extent are zero-filled),
//          and the consumers read every tap out of the same chunk with ldmatrix at a row offset, into registers that feed
//          the RS form of wgmma.  A tap that falls off the board points the lane at a 128-byte row of zeros instead.
//   GEMM   (!CONV): A [M][K] rows, 128 per tile, one smem stage per K block beside B (SS form of wgmma).
// Tile: M_TILE pixels / rows x N_TILE output channels (<= 256), K walks taps x C_in in 64-channel blocks (128-byte swizzled
//   rows), tap outer, channel block inner.  Every output element accumulates its K blocks in the same order whatever the tile
//   shape, so results do not depend on M_TILE, N_TILE or on how the tiles are spread over CTAs.
// CTA = 3 warpgroups: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers, each issuing m64nN wgmma on its
//   M_TILE / 2 rows of the tile (one or two m64 blocks) with fp32 accumulators in registers, then running the epilogue from
//   those registers (+bias (+residual) -> ReLU -> fp16 / fp32 -> HBM).  The B operand (weights) streams through a kStages-deep
//   smem ring with full/empty mbarriers; the conv's A chunks have a full/empty pair each.  The producer runs ahead into the
//   next tile while the consumers store the current one: chunk kc of the next tile loads as soon as every consumer warp has
//   read tap 8 of chunk kc, under the MMAs of the chunks after it.  Persistent: grid <= #SMs, tiles strided over CTAs.
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
constexpr int kTileM = 128;                 // M tile of the GEMM mode and of the conv's small-batch (64-column) form
constexpr int kAStageBytes = kTileM * 128;  // GEMM: 16 KB
constexpr int kThreads = 384;
constexpr int kConsumerWarps = 8;
constexpr int kSmemLimit = 232448;          // opt-in dynamic shared memory per CTA on sm_90 (227 KB)
constexpr int kMaxStages = 8;
constexpr int kEpiCols = 32;                       // columns per step of the staged epilogue
constexpr int kEpiSlotBytes = 64 * kEpiCols * 2;   // 4 KB: 64 rows x 32 fp16
constexpr int kEpiSlots = 3;                       // per consumer warpgroup: one being written, two being stored
constexpr int kEpiBytes = kEpiSlots * kEpiSlotBytes;
// conv A operand: a tap reaches 9 dy + dx = -10 .. +10 rows from its output pixel.  The halo load of a tile is M_TILE / 128
// boxes of kHaloBox rows (a multiple of 8, so every box starts on a 1024-byte swizzle atom, and >= 128 + 2 kHalo).
constexpr int kHalo = 10;
constexpr int kHaloBox = 152;
constexpr int kMaxChunks = 4;               // C_in / 64 <= 4

struct Args {
  int n_taps;        // 9 (3x3 conv) or 1 (plain GEMM)
  int k_chunks;      // C_in / 64
  int tile_m;        // M tile: 128, or 256 for the conv's full-width form (selects the kernel instance)
  int m_tiles;       // ceil(rows / tile_m): the host's grid bound (an upper bound when n_dev is set)
  int n_tiles;       // ceil(N / N_TILE)
  int rows;          // conv: pixels (n_boards*90); GEMM: M
  int n_total;       // B-operand rows per tap (C_out padded to N_TILE multiple)
  int n_valid;       // real number of output columns
  int ldo;           // output leading dimension in elements
  int conv;          // 1: 3x3 conv over [B*90][C] pixels, A loaded once per tile with its halo; 0: GEMM
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

// Shared memory: the conv's A chunks, the operand ring (GEMM: A and B per stage; conv: B), the epilogue ring of both consumer
// warpgroups, barriers and the conv's zero row.  The ring takes as many stages as still fit.
template <int N_TILE, int M_TILE, bool CONV>
struct Cfg {
  static constexpr int kMB = M_TILE / 128;                        // m64 blocks per consumer warpgroup
  static constexpr int kAChunkBytes = kMB * kHaloBox * 128;       // conv: one 64-channel block of the tile's rows + halo
  static constexpr int kABytes = CONV ? kMaxChunks * kAChunkBytes : 0;
  static constexpr int kBStageBytes = N_TILE * 128;
  static constexpr int kStageBytes = (CONV ? 0 : kAStageBytes) + kBStageBytes;
  static constexpr int kMiscBytes = 512;                          // barriers (256 B), then the zero row
  static constexpr int kFit = (kSmemLimit - kABytes - 2 * kEpiBytes - kMiscBytes - 1024) / kStageBytes;
  static constexpr int kStages = kFit > kMaxStages ? kMaxStages : kFit;
  static constexpr int kSmemBytes = kABytes + kStages * kStageBytes + 2 * kEpiBytes + kMiscBytes + 1024;   // + alignment slack
  static_assert(N_TILE % 64 == 0 && N_TILE <= 256, "wgmma N tile");
  static_assert(M_TILE == 128 || (CONV && M_TILE == 256), "M tile");
  static_assert(kMB * N_TILE <= 256, "accumulators: at most 128 fp32 registers per thread");
  static_assert(kMB * kHaloBox >= M_TILE + 2 * kHalo && kHaloBox % 8 == 0 && kHaloBox <= 256, "halo boxes");
  static_assert(kStages >= 2 && kSmemBytes <= kSmemLimit, "shared memory");
  static_assert((2 * kStages + 2 * kEpiSlots + 2 * kMaxChunks) * 8 <= 256, "barrier space");
};

template <int N_TILE, int M_TILE, bool CONV>
__global__ void __launch_bounds__(kThreads, 1)
k_igemm(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
        const Args a) {
  using C = Cfg<N_TILE, M_TILE, CONV>;
  constexpr int S = C::kStages, MB = C::kMB;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sa = smem;                                                         // conv: [kMaxChunks][kAChunkBytes]
  uint8_t* sring = smem + C::kABytes;                                         // [S][kStageBytes]
  uint8_t* epi = sring + S * C::kStageBytes;                                  // [2 warpgroups][kEpiBytes]
  uint64_t* full = reinterpret_cast<uint64_t*>(epi + 2 * kEpiBytes);          // [S]  TMA -> MMA
  uint64_t* empty = full + S;                                                 // [S]  MMA -> TMA (one arrive per consumer warp)
  uint64_t* efree = empty + S;    // [2][kEpiSlots]  the slot's last store has read it: the warpgroup may write it again
  uint64_t* afull = efree + 2 * kEpiSlots;      // [kMaxChunks] conv: the tile's chunk has landed
  uint64_t* aempty = afull + kMaxChunks;        // [kMaxChunks] conv: every consumer warp has read the chunk's last tap
  uint8_t* zrow = epi + 2 * kEpiBytes + 256;    // conv: 128 zero bytes, the A row of a tap that falls off the board

  const int wgi = threadIdx.x >> 7, t = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { wg::mbar_init(&full[s], 1); wg::mbar_init(&empty[s], kConsumerWarps); }
    for (int s = 0; s < 2 * kEpiSlots; ++s) wg::mbar_init(&efree[s], 1);
    for (int s = 0; s < kMaxChunks; ++s) { wg::mbar_init(&afull[s], 1); wg::mbar_init(&aempty[s], kConsumerWarps); }
    wg::fence_barrier_init();
  }
  if (CONV && threadIdx.x < 32) reinterpret_cast<uint32_t*>(zrow)[threadIdx.x] = 0u;
  wg::griddep_launch_dependents();     // (PDL launches only) the next conv may become resident while this one runs
  __syncthreads();
  wg::griddep_wait();                  // (PDL launches only) the producer of this conv's input has completed

  const int n_kb = a.n_taps * a.k_chunks;
  const int rows = args_rows(a);
  const int m_tiles = (rows + M_TILE - 1) / M_TILE;
  const int total_tiles = m_tiles * a.n_tiles;
  // conv: the N tiles of an M tile are neighbours in tile order, so they run side by side and share its halo and skip rows
  // in L2.  GEMM: M tiles first.
  auto tile_mn = [&](int tile, int& m_tile, int& n_tile) {
    if (CONV) { m_tile = tile / a.n_tiles; n_tile = tile % a.n_tiles; }
    else { m_tile = tile % m_tiles; n_tile = tile / m_tiles; }
  };

  constexpr int kSteps = N_TILE / kEpiCols;                // steps of the staged epilogue per m64 block
  auto tile_staged = [&](int m_tile) { return a.staged && m_tile * M_TILE + M_TILE <= rows; };

  if (wgi == 0) {
    // ------------------------------------------------------------ TMA producer
    wg::reg_dealloc<40>();
    if (t == 0) {
      wg::prefetch_tmap(&tmA);
      wg::prefetch_tmap(&tmB);
      // Conv with a skip stream: the epilogue reads the tile's skip rows right after the last MMA, when every CTA of the
      // wave does the same, so the reads would all miss L2 at once with the tensor cores idle.  Halfway through the tile's
      // main loop the producer of N tile 0 prefetches the M tile's whole skip rows (all N tiles; rows below args_rows only)
      // into L2 instead.  Halfway rather than at the tile's first load: the first load is issued while the previous tile's
      // epilogue still has to stream its outputs through L2, which could evict the prefetched lines.
      const uint8_t* skip = !CONV ? nullptr : a.residual32 ? reinterpret_cast<const uint8_t*>(a.residual32)
                                                             : reinterpret_cast<const uint8_t*>(a.residual);
      const int skip_es = a.residual32 ? 4 : 2;
      uint32_t s = 0, ph = 0, aph = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int m_tile, n_tile;
        tile_mn(tile, m_tile, n_tile);
        const int pix0 = m_tile * M_TILE;
        for (int kb = 0; kb < n_kb; ++kb) {
          const int tap = kb / a.k_chunks, kc = kb - tap * a.k_chunks;
          if (skip && n_tile == 0 && kb == n_kb / 2) {
            const int nr = min(M_TILE, rows - pix0);
            wg::prefetch_l2_bulk(skip + (long long)pix0 * a.ldo * skip_es, (uint32_t)(nr * a.ldo * skip_es));
          }
          if (CONV && tap == 0) {              // chunk kc of this tile, once its previous tile has read tap 8 of it
            uint8_t* dst = sa + kc * C::kAChunkBytes;
            wg::mbar_wait(&aempty[kc], aph ^ 1);
            wg::mbar_expect_tx(&afull[kc], (uint32_t)C::kAChunkBytes);
#pragma unroll
            for (int b = 0; b < MB; ++b)
              wg::tma_load_2d(dst + b * kHaloBox * 128, &tmA, &afull[kc], kc * kBlockK, pix0 - kHalo + b * kHaloBox);
          }
          wg::mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = sring + s * C::kStageBytes;
          wg::mbar_expect_tx(&full[s], (uint32_t)C::kStageBytes);
          if (!CONV) wg::tma_load_2d(st, &tmA, &full[s], kc * kBlockK, m_tile * kTileM);
          wg::tma_load_2d(st + (CONV ? 0 : kAStageBytes), &tmB, &full[s], kc * kBlockK, tap * a.n_total + n_tile * N_TILE);
          if (++s == (uint32_t)S) { s = 0; ph ^= 1; }
        }
        aph ^= 1;
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers: MMA + epilogue on rows cw*MB*64 .. +MB*64-1
  wg::reg_alloc<232>();
  const int cw = wgi - 1, warp = t >> 5, lane = t & 31;
  const int mrow = cw * MB * 64 + warp * 16 + (lane >> 2); // accumulator rows mrow + 64 mb and mrow + 64 mb + 8 of the tile
  const int cq = 2 * (lane & 3);                            // first of the two adjacent columns per 8-column group
  float acc[MB][N_TILE / 2];
  // staged epilogue: this warpgroup's slots and barriers; byte offset of this thread's first row (warp * 16 + lane / 4 of the
  // m64 block; the second is 8 rows on, same swizzle phase) and column pair inside a slot, before the swizzle XOR
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
  uint32_t s = 0, ph = 0, aph = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int m_tile, n_tile;
    tile_mn(tile, m_tile, n_tile);
    uint32_t prev = 0;
    if constexpr (CONV) {
      // This lane's ldmatrix row in m64 block mb is tile row rl = cw*MB*64 + 64 mb + warp*16 + lane % 16 (8 channels from
      // 8 * (lane / 16) of each k16 step); bit `tap` of tmask is set when the tap's input pixel is on the board.  A tap that
      // is on the board stays inside the output pixel's own board, so an output row inside the batch only ever reads rows
      // inside the batch or the zero row.  Rows between the device-side batch and the buffer's extent hold stale data
      // (earlier, larger batches); only output rows beyond the batch, which are never stored, can read them.
      int rl[MB];
      uint32_t tmask[MB];
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) {
        rl[mb] = cw * MB * 64 + mb * 64 + warp * 16 + (lane & 15);
        const int p = (m_tile * M_TILE + rl[mb]) % 90, y = p / 9, x = p % 9;
        uint32_t m = 0;
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
          if (yy >= 0 && yy < 10 && xx >= 0 && xx < 9) m |= 1u << tap;
        }
        tmask[mb] = m;
      }
      const uint32_t sa0 = wg::smem_u32(sa), zaddr = wg::smem_u32(zrow), c8 = lane >> 4;
      uint32_t afr[2][MB][2][4];            // A fragments, double-buffered per half K block (k16 steps 0-1 and 2-3)
      int kb = 0;
      for (int tap = 0; tap < 9; ++tap) {
        const int shift = kHalo + 9 * (tap / 3 - 1) + (tap % 3 - 1);
        // per m64 block: the row's address in chunk 0 and the step to the next chunk, or the zero row; the row's swizzle phase
        uint32_t abase[MB], astep[MB], ax[MB];
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) {
          const bool on = (tmask[mb] >> tap) & 1u;
          const uint32_t r = (uint32_t)(rl[mb] + shift);
          abase[mb] = on ? sa0 + r * 128 : zaddr;
          astep[mb] = on ? (uint32_t)C::kAChunkBytes : 0u;
          ax[mb] = on ? (r & 7) : 0u;
        }
        for (int kc = 0; kc < a.k_chunks; ++kc, ++kb) {
          if (tap == 0) wg::mbar_wait(&afull[kc], aph);
          wg::mbar_wait(&full[s], ph);
          const uint64_t db = wg::smem_desc_sw128(wg::smem_u32(sring + s * C::kStageBytes));
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            // the group that last read afr[hf] (the previous half K block of the same parity) has retired: wait<1> below
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
              for (int kk = 0; kk < 2; ++kk) {
                const uint32_t j = (uint32_t)(2 * (2 * hf + kk)) + c8;            // 16-byte column of the 128-byte row
                wg::ldsm_x4(afr[hf][mb][kk], abase[mb] + kc * astep[mb] + ((j ^ ax[mb]) << 4));
              }
            wg::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 2; ++kk)
#pragma unroll
              for (int mb = 0; mb < MB; ++mb)
                wg::WgmmaRS<N_TILE>::mma(acc[mb], afr[hf][mb][kk], db + (uint64_t)(2 * (2 * hf + kk)), (kb | (2 * hf + kk)) != 0);
            wg::wgmma_commit();
            // the last tap of this chunk is in registers: the producer may load the next tile's chunk over it
            if (hf == 1 && tap == 8 && lane == 0) wg::mbar_arrive(&aempty[kc]);
            wg::wgmma_wait<1>();
            // half 0: the previous K block's groups are done: hand its B stage back to the producer
            if (hf == 0 && kb > 0 && lane == 0) wg::mbar_arrive(&empty[prev]);
          }
          prev = s;
          if (++s == (uint32_t)S) { s = 0; ph ^= 1; }
        }
      }
      aph ^= 1;
    } else {
      for (int kb = 0; kb < n_kb; ++kb) {
        wg::mbar_wait(&full[s], ph);
        const uint32_t sA = wg::smem_u32(sring + s * C::kStageBytes);
        const uint64_t da = wg::smem_desc_sw128(sA + cw * 64 * 128);
        const uint64_t db = wg::smem_desc_sw128(sA + kAStageBytes);
        wg::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k)              // +32 B per k16 step inside the swizzle atom
          wg::Wgmma<N_TILE>::mma(acc[0], da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb | k) != 0);
        wg::wgmma_commit();
        wg::wgmma_wait<1>();                                // the previous stage's MMAs are done: hand it back to the producer
        if (kb > 0 && lane == 0) wg::mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == (uint32_t)S) { s = 0; ph ^= 1; }
      }
    }
    wg::wgmma_wait<0>();
    if (lane == 0) wg::mbar_arrive(&empty[prev]);

    // ------------------------------------------------------------ epilogue
    const int nb = n_tile * N_TILE + cq;                    // column of acc[mb][4j + 2h] is nb + 8j
    if (a.bias) {
#pragma unroll
      for (int j = 0; j < N_TILE / 8; ++j) {                // bias arrays are padded to the N tile
        const float2 b = __ldg(reinterpret_cast<const float2*>(a.bias + nb + 8 * j));
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) {
          acc[mb][4 * j] += b.x; acc[mb][4 * j + 1] += b.y; acc[mb][4 * j + 2] += b.x; acc[mb][4 * j + 3] += b.y;
        }
      }
    }
    if (tile_staged(m_tile)) {
      if (t == 0) { wg::bulk_wait_group_read<0>(); release_to(e_issued); }    // the previous tile's last slots
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) {
#pragma unroll
        for (int st = 0; st < kSteps; ++st) {
          uint8_t* slot = ering + e_slot * kEpiSlotBytes;
          wg::mbar_wait(&fre[e_slot], e_ph ^ 1);            // passes on a slot that has not been used yet
#pragma unroll
          for (int jj = 0; jj < kEpiCols / 8; ++jj) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int i = 4 * (st * (kEpiCols / 8) + jj) + 2 * h;
              float x0 = acc[mb][i], x1 = acc[mb][i + 1];
              if (a.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
              *reinterpret_cast<__half2*>(slot + e_off + h * 8 * 64 + ((jj ^ e_x) << 4)) = __floats2half2_rn(x0, x1);
            }
          }
          wg::fence_proxy_async();
          wg::named_barrier(1 + cw, 128);
          if (t == 0) {
            wg::tma_store_2d(&tmOut, slot, n_tile * N_TILE + st * kEpiCols, m_tile * M_TILE + cw * MB * 64 + mb * 64);
            wg::bulk_commit();
            ++e_issued;
            // hand back the previous step's slot (its store has had this step's time to read it); this step's store stays in flight
            wg::bulk_wait_group_read<1>();
            release_to(e_issued - 1);
          }
          if (++e_slot == kEpiSlots) { e_slot = 0; e_ph ^= 1; }
        }
      }
      continue;
    }
    // accumulator row mrow + 64 mb + 8h: global output row (pixel / GEMM row), and whether it is inside the batch
    auto out_row = [&](int mb, int h, long long& grow, bool& valid) {
      grow = (long long)m_tile * M_TILE + mrow + 64 * mb + 8 * h;
      valid = grow < rows;
    };
    // + skip stream, for all of the thread's rows before the first output store.  The compiler keeps every load behind the
    // stores that precede it (a store might alias the skip stream), so loads interleaved with the stores would go out one
    // round trip at a time; here they go out back to back.  Same operations in the same order: (acc + bias) + skip.
    if (!a.out_f32 && (a.residual32 || a.residual)) {
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          long long grow;
          bool valid;
          out_row(mb, h, grow, valid);
          if (!valid) continue;
          if (a.residual32) {
            const float* r32 = a.residual32 + grow * a.ldo;
#pragma unroll
            for (int j = 0; j < N_TILE / 8; ++j) {
              const float2 r = __ldg(reinterpret_cast<const float2*>(r32 + nb + 8 * j));
              acc[mb][4 * j + 2 * h] += r.x; acc[mb][4 * j + 2 * h + 1] += r.y;
            }
          } else {
            const __half* r16 = a.residual + grow * a.ldo;
#pragma unroll
            for (int j = 0; j < N_TILE / 8; ++j) {
              const float2 r = __half22float2(__ldg(reinterpret_cast<const __half2*>(r16 + nb + 8 * j)));
              acc[mb][4 * j + 2 * h] += r.x; acc[mb][4 * j + 2 * h + 1] += r.y;
            }
          }
        }
      }
    }
#pragma unroll
    for (int mb = 0; mb < MB; ++mb) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        long long grow;                                     // global output row
        bool valid;
        out_row(mb, h, grow, valid);
        if (a.out_f32) {
          if (a.row_stats) {                                // the 4 threads of a quad hold one row: reduce across them
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < N_TILE / 8; ++j) {
              if (nb + 8 * j < a.n_valid) mx = fmaxf(mx, acc[mb][4 * j + 2 * h]);
              if (nb + 8 * j + 1 < a.n_valid) mx = fmaxf(mx, acc[mb][4 * j + 2 * h + 1]);
            }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            float sum = 0.f;
#pragma unroll
            for (int j = 0; j < N_TILE / 8; ++j) {
              if (nb + 8 * j < a.n_valid) sum += __expf(acc[mb][4 * j + 2 * h] - mx);
              if (nb + 8 * j + 1 < a.n_valid) sum += __expf(acc[mb][4 * j + 2 * h + 1] - mx);
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
            float x0 = acc[mb][4 * j + 2 * h], x1 = acc[mb][4 * j + 2 * h + 1];
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
            float x0 = acc[mb][4 * j + 2 * h], x1 = acc[mb][4 * j + 2 * h + 1];
            if (a.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
            *reinterpret_cast<__half2*>(o + n) = __floats2half2_rn(x0, x1);
            if (o32) *reinterpret_cast<float2*>(o32 + n) = make_float2(x0, x1);
          }
        }
      }
    }
  }
  if (t == 0) wg::bulk_wait_group_all();                    // the staged stores have landed before the grid can count as complete
}

}  // namespace igemm
