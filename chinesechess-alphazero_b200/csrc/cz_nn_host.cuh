// cz_nn_host.cuh — host helpers of the network runtime (cz_nn.cu) shared with the trainer (cz_train.cu): tensor-map
// builders and the k_igemm launcher.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

namespace igemm { struct Args; }

namespace cznn {

// fp16 NHWC activations [n_images][10][9][c] in im2col mode for a 3x3 "same" convolution, 64 channels x `pixels` per load
int make_map_im2col(CUtensorMap* m, const void* base, int c, long long n_images, int pixels = 128);
// fp16 matrix [rows][k] (k contiguous), box {64, box_rows}, 128-byte swizzle, zero OOB fill
int make_map_2d(CUtensorMap* m, const void* base, int k, long long rows, int box_rows);
int num_sms();
// igemm::k_igemm<n_tile> on `st` (n_tile 64 / 128 / 192 / 256).  `out_map`: tensor map of a.out for the staged epilogue of a
// dense conv with fp16 output and no skip stream (Args::staged is set from it); null: register epilogue.
int launch_igemm(int n_tile, const CUtensorMap& tmA, const CUtensorMap& tmB, const igemm::Args& a, cudaStream_t st,
                 const CUtensorMap* out_map = nullptr);

}  // namespace cznn
