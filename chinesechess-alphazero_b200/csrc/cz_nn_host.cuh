// cz_nn_host.cuh — host helpers of the network runtime (cz_nn.cu) shared with the trainer (cz_train.cu): error macro,
// workspace carver, Keras tensor lookup, tensor-map builders, the conv's k_igemm arguments and the k_igemm launcher.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <string>

#include "cz_err.h"
#include "../../include/cczero_b200.h"

#define CZ_CUDA(x)                                                                           \
  do {                                                                                       \
    cudaError_t e__ = (x);                                                                   \
    if (e__ != cudaSuccess) return cz_fail(CZ_ERR_CUDA, "%s: %s", #x, cudaGetErrorString(e__)); \
  } while (0)

namespace igemm { struct Args; }

namespace cznn {

// Hands out 1 KB-aligned ranges of a workspace in call order; with base = null it only counts (off = bytes needed).
struct Carver {
  uint8_t* base; size_t off;
  void* take(size_t bytes) {
    off = (off + 1023) & ~(size_t)1023;
    void* p = base ? base + off : nullptr;
    off += bytes;
    return p;
  }
};

// The tensor of descs[0, n) named "<layer>[-k-f]/<weight>[:0]" (Keras appends "-<k>-<f>" to conv layer names and ":0" to
// weights; "<layer>/<layer>/<weight>" is accepted too), or null.
const cz_tensor_desc* find_keras_tensor(const cz_tensor_desc* descs, int n, const std::string& layer, const std::string& weight);

// fp16 NHWC activations [n_images][10][9][c] in im2col mode for a 3x3 "same" convolution, 64 channels x `pixels` per load
// (the weight gradient's operand)
int make_map_im2col(CUtensorMap* m, const void* base, int c, long long n_images, int pixels);
// fp16 matrix [rows][k] (k contiguous), box {64, rows_per_box}, 128-byte swizzle, zero OOB fill
int make_map_2d(CUtensorMap* m, const void* base, int k, long long rows, int rows_per_box);
int num_sms();
// k_igemm arguments of a 3x3 "same" conv over fp16 activations [n_boards*90][c]: out = relu?(conv + bias (+ residual)),
// fp16 out of the same layout; bias and residual may be null.  The caller adds a device-side batch, a skip stream or fp32 out.
// `split`: the small-batch form, 64-column tiles.  The launch takes N tile conv_tile_n(c, split), the weights' tensor map
// boxes of that many rows and the input's map from make_map_2d(..., igemm::kHaloBox).
igemm::Args conv_args(int n_boards, int c, const float* bias, const __half* residual, void* out, int relu, bool split = false);
int conv_tile_n(int c, bool split);
// igemm::k_igemm<n_tile> on `st` (n_tile 64 / 128 / 192 / 256) with programmatic dependent launch.  `out_map`: tensor map of
// a.out for the staged epilogue of a conv with fp16 output and no skip stream (Args::staged is set from it); null: register
// epilogue.
int launch_igemm(int n_tile, const CUtensorMap& tmA, const CUtensorMap& tmB, const igemm::Args& a, cudaStream_t st,
                 const CUtensorMap* out_map = nullptr);

}  // namespace cznn
