// cz_nn.cuh — interface between the search engine and the network runtime (cz_nn.cu).
#pragma once
#include <stdint.h>
#include <stddef.h>
#include "../../include/cczero_b200.h"

namespace cznn {

struct NnRuntime;

// bytes of device workspace the runtime needs for batches up to max_batch positions
// pol_c / val_c: channels of the policy / value 1x1 convolutions (0 = agent/model.py's 4 / 2)
size_t nn_workspace_bytes(int filters, int blocks, int value_fc, int max_batch, int n_nets, int pol_c, int val_c);
// returns nullptr and sets cz_last_error on failure
NnRuntime* nn_create(int device, int filters, int blocks, int value_fc, int max_batch, void* workspace, size_t bytes,
                     void* stream, int fp32_skip_mode, int n_nets, int in_planes /* 14 or 28 */, int pol_c, int val_c);
void nn_destroy(NnRuntime*);
int nn_set_weights(NnRuntime*, int net, const cz_tensor_desc* descs, int n);
bool nn_ready(const NnRuntime*);
// boards_dev: [batch][96] packed boards ([batch][2][96] = board, history board when in_planes = 28); policy_dev [batch][2086] f32 softmax; value_dev [batch] f32
int nn_forward_boards(NnRuntime*, int net, const uint8_t* boards_dev, int batch, float* policy_dev, float* value_dev);
int nn_forward_planes(NnRuntime*, int net, const float* planes_dev, int batch, float* policy_dev, float* value_dev);
// Evaluation step of the integrated search: at most n_max leaves, the actual count is the DEVICE integer *n_dev (fixed launch
// shapes, capturable into a CUDA graph).  labels_dev [n][CZ_MAX_MOVES] int16 = action label of every legal move (-1: none),
// label_counts_dev [n]; legal_p_dev [n][CZ_MAX_MOVES] f32 gets the softmax probability of exactly those labels — bit for bit
// the numbers nn_forward_boards writes at those indices of its [n][2086] vector.
// Mirror form (mirror_lut_dev = cz_mirror_labels on the device, value2_dev [2 * n_max] scratch): boards_dev holds the n
// leaves and then their mirrors, n_dev[2] = 2 * n_dev[0] rows are evaluated, and leaf i gets
// 0.5 * (p_i[lab] + p_{n+i}[M lab]) and 0.5 * (v_i + v_{n+i}), each sum and product rounded once in fp32.
int nn_forward_leaves(NnRuntime*, int net, const uint8_t* boards_dev, int n_max, const int* n_dev, const int16_t* labels_dev,
                      const int32_t* label_counts_dev, float* legal_p_dev, float* value_dev,
                      const int16_t* mirror_lut_dev, float* value2_dev);
bool nn_profiling(const NnRuntime*);
// launches of one nn_forward_leaves, the two profiling stamps included while profiling is on
int nn_launches_per_forward(const NnRuntime*);
uint64_t nn_launches(const NnRuntime*);
// While on, every forward brackets its residual tower with two stamp kernels (capturable, like the rest of the forward).
void nn_profile(NnRuntime*, bool on);
int nn_profile_read(NnRuntime*, double* ms, uint64_t* launches, double* flops);
// cz_nn_read_buffer (include/cczero_b200.h): rows of an intermediate buffer of the last forward; synchronises
int nn_read_buffer(NnRuntime*, int which, int n, void* dst_dev, long long dst_bytes, long long* row_bytes);

}  // namespace cznn
