// cz_simt.h — warp-level primitives used by every integer (board / tree) kernel.
//
// The kernels are written warp-per-game: 32 lanes cooperate on one board or one
// search tree, control flow around every collective is warp-uniform, and there is
// no inter-warp communication.  On the device (nvcc, sm_90a) the primitives map
// 1:1 to __shfl_sync / __ballot_sync / __syncwarp.  With -DCZ_EMUL the very same
// kernel source is compiled by g++ against tests/simt_emul/ (32 fibers per warp on
// one OS thread) so the CPU-only test tier can single-step device logic.  The
// emulator is TEST INFRASTRUCTURE: the shipped library (libcczero_b200.so) is
// always the nvcc build and has no CPU path.
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(CZ_EMUL)
// ---------------------------------------------------------------- CPU emulation
#include <math.h>
#include <string.h>
#define CZ_D static inline
#define CZ_DN static
#define CZ_DM inline
#define CZ_HD static inline
#define CZ_KERNEL(name) void name
#define CZ_RESTRICT __restrict__

struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };

namespace czs {
struct EmulWarp;                       // tests/simt_emul/simt_emul.cpp
extern thread_local int  tl_lane;      // lane id of the running fiber
extern thread_local int  tl_warp;      // warp index inside the block
extern thread_local int  tl_nwarps;    // warps per block
extern thread_local int  tl_block;     // blockIdx.x
extern thread_local unsigned char* tl_smem;  // dynamic shared memory of the block
unsigned emul_ballot(bool p);
uint64_t emul_shfl64(uint64_t v, int src);
void     emul_sync();

CZ_D int lane() { return tl_lane; }
CZ_D int warp_in_block() { return tl_warp; }
CZ_D int warps_per_block() { return tl_nwarps; }
CZ_D int block_idx() { return tl_block; }
CZ_D unsigned char* dyn_smem() { return tl_smem; }
CZ_D unsigned ballot(bool p) { return emul_ballot(p); }
CZ_D void syncwarp() { emul_sync(); }
template <class T> CZ_D T shfl(T v, int src) {
  static_assert(sizeof(T) <= 8, "shfl payload");
  uint64_t u = 0; memcpy(&u, &v, sizeof(T));
  u = emul_shfl64(u, src & 31);
  T r; memcpy(&r, &u, sizeof(T)); return r;
}
CZ_D int popc(unsigned x) { return __builtin_popcount(x); }
CZ_D int ffs(unsigned x) { return __builtin_ffs((int)x); }          // 1-based, 0 if none
CZ_D int fls(unsigned x) { return x ? 32 - __builtin_clz(x) : 0; }  // 1-based msb, 0 if none
CZ_D int nth_set_bit(unsigned x, int n) {                            // position of the n-th (0-based) set bit, -1 if none
  for (int i = 0; i < 32; ++i) if ((x >> i) & 1u) { if (n == 0) return i; --n; }
  return -1;
}
CZ_D double dsqrt(double x) { return sqrt(x); }
// fast single-precision transcendentals of the root-noise sampler (statistical parity only, never bit-compared)
CZ_D float flog(float x) { return logf(x); }
CZ_D float fcos(float x) { return cosf(x); }
CZ_D float fpow(float x, float y) { return powf(x, y); }
CZ_D float fsqrt(float x) { return sqrtf(x); }
template <class T> CZ_D T ldg(const T* p) { return *p; }
}  // namespace czs

#else
// ---------------------------------------------------------------- device (nvcc)
#include <cuda_runtime.h>
#define CZ_D __device__ __forceinline__
// Big, multiply-called rules functions are real calls on the device: inlined at every site the search kernel grew to 33 k SASS
// instructions (527 KB), far beyond the instruction cache (ncu: 12 % of its issue slots waited for instruction fetch).
#define CZ_DN static __device__ __noinline__
#define CZ_DM __device__ __forceinline__
#define CZ_HD __host__ __device__ __forceinline__
#define CZ_KERNEL(name) __global__ void name
#define CZ_RESTRICT __restrict__

namespace czs {
CZ_D int lane() { return threadIdx.x & 31; }
CZ_D int warp_in_block() { return threadIdx.x >> 5; }
CZ_D int warps_per_block() { return blockDim.x >> 5; }
CZ_D int block_idx() { return blockIdx.x; }
CZ_D unsigned char* dyn_smem() { extern __shared__ __align__(16) unsigned char cz_dyn_smem[]; return cz_dyn_smem; }
CZ_D unsigned ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
CZ_D void syncwarp() { __syncwarp(); }
template <class T> CZ_D T shfl(T v, int src) { return __shfl_sync(0xffffffffu, v, src); }
CZ_D int popc(unsigned x) { return __popc(x); }
CZ_D int ffs(unsigned x) { return __ffs((int)x); }
CZ_D int fls(unsigned x) { return 32 - __clz((int)x); }
CZ_D int nth_set_bit(unsigned x, int n) { const unsigned r = __fns(x, 0u, n + 1); return r == 0xffffffffu ? -1 : (int)r; }
CZ_D double dsqrt(double x) { return __dsqrt_rn(x); }
CZ_D float flog(float x) { return __logf(x); }
CZ_D float fcos(float x) { return __cosf(x); }
CZ_D float fpow(float x, float y) { return __powf(x, y); }
CZ_D float fsqrt(float x) { return __fsqrt_rn(x); }
template <class T> CZ_D T ldg(const T* p) { return __ldg(p); }
}  // namespace czs
#endif

namespace czs {
// ---- collectives built on the primitives (identical on both builds) ----------
CZ_D bool any(bool p) { return ballot(p) != 0u; }
CZ_D bool all(bool p) { return ballot(p) == 0xffffffffu; }

template <class T> CZ_D T shfl_xor(T v, int m) { return shfl(v, lane() ^ m); }

CZ_D int warp_sum(int v) {
  for (int m = 16; m; m >>= 1) v += shfl_xor(v, m);
  return v;
}
CZ_D uint64_t warp_xor64(uint64_t v) {
  for (int m = 16; m; m >>= 1) v ^= shfl_xor(v, m);
  return v;
}
// exclusive prefix sum of a small non-negative int; *total gets the warp sum
CZ_D int warp_excl_scan(int v, int* total) {
  int x = v;
  for (int d = 1; d < 32; d <<= 1) {
    int y = shfl(x, lane() - d);
    if (lane() >= d) x += y;
  }
  *total = shfl(x, 31);
  return x - v;
}
}  // namespace czs
