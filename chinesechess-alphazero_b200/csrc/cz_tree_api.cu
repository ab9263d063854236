// cz_tree_api.cu — the search engine object behind the C-ABI: workspace carving, kernels (one warp per
// game), and the cz_search_* / cz_get_root entry points.  Builds with nvcc (product) or g++ -DCZ_EMUL
// (CPU test tier; the network is unavailable there and only the external-evaluator path works).
#include "../../include/cczero_b200.h"
#include "cz_tree.cuh"
#include "cz_selfplay.cuh"
#include "cz_rt.h"
#include "cz_err.h"
#if !defined(CZ_EMUL)
#include "cz_nn.cuh"
#endif
#include <stdlib.h>
#include <new>
#include <vector>

using namespace cz;

namespace {

constexpr int kWarps = 4;   // games per block

CZ_D TreeSmem* tree_smem() { return reinterpret_cast<TreeSmem*>(czs::dyn_smem()) + czs::warp_in_block(); }
CZ_D int my_game() { return czs::block_idx() * czs::warps_per_block() + czs::warp_in_block(); }

CZ_KERNEL(k_begin)(EngineDev E, int sims_override, int raw_tasks) {
  const int g = my_game();
  if (g >= E.n_games) return;
  game_begin(E, g, sims_override, raw_tasks != 0, tree_smem());
}
// more simulations for the search cz_search_begin opened (same root options, noise table position and counters)
CZ_KERNEL(k_more)(EngineDev E, int n_sims) {
  const int g = my_game();
  if (g >= E.n_games) return;
  if (czs::lane() == 0 && E.active[g]) { E.tasks_left[g] = n_sims; E.round_pending[g] = 0; }
}
CZ_KERNEL(k_pv)(EngineDev E, int g, int max_len, cz_pv_info* out) {
  float v; int has;
  const int len = game_pv(E, g, max_len, out->moves, &v, &has, tree_smem());
  if (czs::lane() == 0) { out->n_moves = len; out->value = v; out->has_value = has; }
}
// The search kernels work on a game range [g0, g1): in arena mode the device-driven loop evaluates each half of the games
// with its own network.  Per-game results do not depend on the split.
CZ_KERNEL(k_wave)(EngineDev E, int g0, int g1) {
  const int g = g0 + my_game();
  if (g >= g1) return;
  game_wave(E, g, tree_smem());
}
CZ_KERNEL(k_apply)(EngineDev E, int g0, int g1, const float* policy, const float* legal_p, const float* value) {
  const int g = g0 + my_game();
  if (g >= g1) return;
  game_apply(E, g, policy, legal_p, value, tree_smem());
}
// device-driven loop: the same warp applies the evaluation of the previous wave and walks the next one (the game's state stays hot)
CZ_KERNEL(k_apply_wave)(EngineDev E, int g0, int g1, const float* legal_p, const float* value) {
  const int g = g0 + my_game();
  if (g >= g1) return;
  TreeSmem* sm = tree_smem();
  game_apply(E, g, nullptr, legal_p, value, sm);
  czs::syncwarp();
  game_wave(E, g, sm);
}
// single warp: exclusive scan of the per-game leaf counts, totals[0] = leaves, totals[1] = any game busy
CZ_KERNEL(k_scan)(EngineDev E, int gb, int ge, int slot) {
  int base = 0, busy = 0;
  for (int g0 = gb; g0 < ge; g0 += 32) {
    const int g = g0 + czs::lane();
    const int n = g < ge ? E.n_leaf[g] : 0;
    int tot;
    const int off = czs::warp_excl_scan(n, &tot);
    if (g < ge) {
      E.leaf_off[g] = base + off;                      // offset inside this slot's dense list
      if (E.active[g] && (E.round_pending[g] > 0 || E.tasks_left[g] > 0)) busy = 1;
    }
    base += tot;
  }
  busy = czs::any(busy != 0) ? 1 : 0;
  if (czs::lane() == 0) {
    E.totals[4 * slot] = base; E.totals[4 * slot + 1] = busy;
#if defined(CZ_EMUL)
    E.counters[1] += (unsigned long long)base; E.counters[2] += 1;        // positions sent to the evaluator, wave iterations
#else
    atomicAdd(E.counters + 1, (unsigned long long)base); atomicAdd(E.counters + 2, 1ULL);
#endif
  }
}
// dense leaf list of a range: boards, and the action labels of each leaf's legal moves in edge order, which is all the
// evaluation step has to know to hand back exactly the priors the search will read
#if !defined(CZ_EMUL)
// The same scan with one thread per game (1024 threads, chunked): the single-warp version walks 32 dependent chunks at
// 1024 games (52 us in the c3 launch list); this one is a couple of microseconds.  Same outputs, same counters.
__global__ void __launch_bounds__(1024) k_scan_block(EngineDev E, int gb, int ge, int slot) {
  __shared__ int warp_tot[32];
  __shared__ int carry_s, busy_s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { carry_s = 0; busy_s = 0; }
  __syncthreads();
  for (int g0 = gb; g0 < ge; g0 += 1024) {
    const int g = g0 + tid;
    const int n = g < ge ? E.n_leaf[g] : 0;
    int x = n;
    for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) warp_tot[warp] = x;
    if (g < ge && E.active[g] && (E.round_pending[g] > 0 || E.tasks_left[g] > 0)) busy_s = 1;     // benign race: all writers store 1
    __syncthreads();
    int wbase = 0;
    for (int w = 0; w < warp; ++w) wbase += warp_tot[w];
    const int carry = carry_s;
    if (g < ge) E.leaf_off[g] = carry + wbase + x - n;
    __syncthreads();
    if (tid == 1023) carry_s = carry + wbase + x;
    __syncthreads();
  }
  if (tid == 0) {
    const int base = carry_s;
    E.totals[4 * slot] = base; E.totals[4 * slot + 1] = busy_s;
    atomicAdd(E.counters + 1, (unsigned long long)base); atomicAdd(E.counters + 2, 1ULL);
  }
}
#endif
// mirror_tot (eval_mirror, device-driven loop): the range's totals slot; leaf j of the range is also written, mirrored, at
// row totals[0] + j, and totals[2] = 2 * totals[0] is the row count the network reads.  Null: the plain form.
CZ_KERNEL(k_gather)(EngineDev E, int g0, int g1, uint8_t* dense, int16_t* labels, int32_t* nlab, int32_t* mirror_tot) {
  const int g = g0 + my_game();
  if (g >= g1) return;
  const int n_range = mirror_tot ? mirror_tot[0] : 0;
  if (mirror_tot && g == g0 && czs::lane() == 0) mirror_tot[2] = 2 * n_range;
  const int n = E.n_leaf[g], off = E.leaf_off[g];
  for (int j = 0; j < n; ++j) {
    const uint8_t* s = E.leaf_board + ((size_t)g * E.K + j) * E.lb_stride;
    uint8_t* d = dense + (size_t)(off + j) * E.lb_stride;
    if (czs::lane() < E.lb_stride / 16) reinterpret_cast<uint4*>(d)[czs::lane()] = reinterpret_cast<const uint4*>(s)[czs::lane()];
    if (mirror_tot)
      for (int b = 0; b < E.lb_stride; b += BOARD_STRIDE) mirror_board(s + b, dense + (size_t)(n_range + off + j) * E.lb_stride + b);
    const int node = E.sim_leaf_node[(size_t)g * E.K + E.leaf_sim[(size_t)g * E.K + j]];
    const size_t ni = (size_t)g * E.ncap + node;
    const int L = (int)(E.node_meta[ni] & 0xff);
    const size_t eo = (size_t)g * E.ecap + E.node_edge_off[ni];
    for (int i = czs::lane(); i < L; i += 32) {
      const move_t m = E.edge_move[eo + i];
      labels[(size_t)(off + j) * MAX_MOVES + i] = E.label_lut[mv_from(m) * 90 + mv_to(m)];
    }
    if (czs::lane() == 0) nlab[off + j] = L;
  }
}
// Device-driven search loop, end of an iteration: count it in *iters (mapped pinned memory, read by the host after the
// search's synchronise for cz_launch_count) and, inside the WHILE node's body, run the body again while any range has work.
CZ_KERNEL(k_loop_flag)(EngineDev E, int n_slots, int32_t* iters, unsigned long long cond_handle, int set_cond) {
  if (czs::lane() != 0) return;
  int busy = 0;
  for (int s = 0; s < n_slots; ++s) busy |= (E.totals[4 * s] > 0) | (E.totals[4 * s + 1] != 0);
  const int it = E.loop_iter[0] + 1;
  E.loop_iter[0] = it;
  *iters = it;
#if !defined(CZ_EMUL)
  if (set_cond) cudaGraphSetConditional((cudaGraphConditionalHandle)cond_handle, busy ? 1u : 0u);
#else
  (void)cond_handle; (void)set_cond;
#endif
}
CZ_KERNEL(k_loop_reset)(EngineDev E) {
  if (czs::lane() == 0) { E.loop_iter[0] = 0; for (int i = 0; i < 8; ++i) E.totals[i] = 0; }
}
CZ_KERNEL(k_planes_dense)(const uint8_t* boards, int n, float* planes, int lb_stride) {
  const int i = my_game();
  if (i >= n) return;
  TreeSmem* sm = tree_smem();
  const int n_boards = lb_stride / BOARD_STRIDE;             // 2 with use_history: planes 14-27 = the history board
  for (int h = 0; h < n_boards; ++h) {
    copy_board(boards + (size_t)i * lb_stride + h * BOARD_STRIDE, sm->board);
    encode_planes_f32(sm->board, planes + ((size_t)i * n_boards + h) * 14 * NSQ);
    czs::syncwarp();
  }
}
CZ_KERNEL(k_reset)(EngineDev E, const uint8_t* boards /* [G][96] or null */, const uint8_t* init_board, int clear_game /* -1 all */) {
  const int g = my_game();
  if (g >= E.n_games) return;
  if (clear_game >= 0 && g != clear_game) return;
  const uint8_t* src = boards ? boards + (size_t)g * BOARD_STRIDE : init_board;
  for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) E.root_board[(size_t)g * BOARD_STRIDE + k] = k < NSQ ? src[k] : (uint8_t)0;
  uint32_t* h = E.hash + (size_t)g * E.hcap;
  for (int i = czs::lane(); i < E.hcap; i += 32) h[i] = 0;
  if (czs::lane() == 0) {
    E.n_nodes[g] = 0; E.n_edges[g] = 0; E.root_node[g] = -1;
    E.tasks_left[g] = 0; E.round_pending[g] = 0; E.n_leaf[g] = 0; E.n_park[g] = 0; E.n_resume[g] = 0;
    E.sims_run[g] = 0; E.noise_used[g] = 0; E.noise_epoch[g] = 0; E.game_err[g] = 0; E.n_no_act[g] = 0; E.increase_temp[g] = 0; E.active[g] = 1;
    E.root_has_hist[g] = 0;
  }
  czs::syncwarp();
  selfplay_reset_game(E, g);
}
CZ_KERNEL(k_set_root)(EngineDev E, int game, const uint8_t* board) {
  for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) E.root_board[(size_t)game * BOARD_STRIDE + k] = k < NSQ ? board[k] : (uint8_t)0;
}
CZ_KERNEL(k_root_info)(EngineDev E, int g, cz_root_info* out) {
  TreeSmem* sm = tree_smem();
  copy_board(E.root_board + (size_t)g * BOARD_STRIDE, sm->board);
  uint64_t k0, k1;
  board_key(sm->board, &k0, &k1);
  const int root = tt_lookup(E, g, k0, k1);
  int L = 0;
  if (root >= 0) {
    const size_t ni = (size_t)g * E.ncap + root;
    L = (int)(E.node_meta[ni] & 0xff);
    const size_t eo = (size_t)g * E.ecap + E.node_edge_off[ni];
    for (int i = czs::lane(); i < L; i += 32) {
      out->moves[i] = E.edge_move[eo + i]; out->n[i] = E.edge_n[eo + i]; out->w[i] = E.edge_w[eo + i]; out->p[i] = E.edge_p[eo + i];
    }
    if (czs::lane() == 0) out->sum_n = E.node_sum_n[ni];
  } else if (czs::lane() == 0) out->sum_n = 0;
  if (czs::lane() == 0) { out->n_moves = L; out->noise_used = E.noise_used[g]; out->sims_run = E.sims_run[g]; }
}
// visit counts of every root (the policy target the trainer consumes, calc_policy player.py:384-385)
CZ_KERNEL(k_root_stats)(EngineDev E, int32_t* n_out, uint16_t* mv_out, int32_t* cnt_out) {
  const int g = my_game();
  if (g >= E.n_games) return;
  const int root = E.root_node[g];
  int L = 0;
  if (root >= 0) {
    const size_t ni = (size_t)g * E.ncap + root;
    L = (int)(E.node_meta[ni] & 0xff);
    const size_t eo = (size_t)g * E.ecap + E.node_edge_off[ni];
    for (int i = czs::lane(); i < MAX_MOVES; i += 32) {
      n_out[(size_t)g * MAX_MOVES + i] = i < L ? E.edge_n[eo + i] : 0;
      mv_out[(size_t)g * MAX_MOVES + i] = i < L ? E.edge_move[eo + i] : (uint16_t)0xFFFF;
    }
  }
  if (czs::lane() == 0) cnt_out[g] = L;
}
CZ_KERNEL(k_set_roots)(EngineDev E, const uint8_t* boards) {
  const int g = my_game();
  if (g >= E.n_games) return;
  for (int k = czs::lane(); k < BOARD_STRIDE; k += 32)
    E.root_board[(size_t)g * BOARD_STRIDE + k] = k < NSQ ? boards[(size_t)g * BOARD_STRIDE + k] : (uint8_t)0;
}
// test hook: draws of the on-device root-noise sampler (noise_mode 1)
CZ_KERNEL(k_noise_sample)(EngineDev E, int game, int n_moves, int count, double* out) {
  for (int i = czs::block_idx() * 32 + czs::lane(); i < count; i += 32 * 64) out[i] = dirichlet_first(E, game, (uint32_t)i, n_moves);
}
// single warp: counters[6] = OR of the per-game error flags, counters[7] = games with any flag set
CZ_KERNEL(k_err_reduce)(EngineDev E) {
  int orv = 0, cnt = 0;
  for (int g = czs::lane(); g < E.n_games; g += 32) { const int f = E.game_err[g]; orv |= f; cnt += f != 0; }
  for (int m = 16; m; m >>= 1) { orv |= czs::shfl_xor(orv, m); cnt += czs::shfl_xor(cnt, m); }
  if (czs::lane() == 0) { E.counters[6] = (unsigned long long)orv; E.counters[7] = (unsigned long long)cnt; }
}
// single warp: sums of the per-game search statistics; out[4] = edges of the nodes currently stored, out[5] = those nodes
CZ_KERNEL(k_stat_reduce)(EngineDev E, unsigned long long* out) {
  unsigned long long a[6] = {0, 0, 0, 0, 0, 0};
  for (int g = czs::lane(); g < E.n_games; g += 32) {
    for (int k = 0; k < 4; ++k) a[k] += E.stat[(size_t)g * 4 + k];
    a[4] += (unsigned long long)E.n_edges[g]; a[5] += (unsigned long long)E.n_nodes[g];
  }
  for (int k = 0; k < 6; ++k) {
    uint32_t lo = (uint32_t)a[k], hi = (uint32_t)(a[k] >> 32);
    for (int m = 16; m; m >>= 1) {
      const unsigned long long o = ((unsigned long long)czs::shfl_xor(hi, m) << 32) | czs::shfl_xor(lo, m);
      a[k] += o; lo = (uint32_t)a[k]; hi = (uint32_t)(a[k] >> 32);
    }
    if (czs::lane() == 0) out[k] = a[k];
  }
}
CZ_KERNEL(k_compact)(EngineDev E) {
  const int g = my_game();
  if (g >= E.n_games) return;
  TreeSmem* sm = tree_smem();
  copy_board(E.root_board + (size_t)g * BOARD_STRIDE, sm->board);
  uint64_t k0, k1;
  board_key(sm->board, &k0, &k1);
  const int root = tt_lookup(E, g, k0, k1);
  if (root >= 0) {
    const int nr = game_compact(E, g, root);
    if (czs::lane() == 0) E.root_node[g] = nr;
  } else {
    clear_tree(E, g);
  }
}
CZ_KERNEL(k_set_noise)(EngineDev E, NoiseRef r) {
  if (czs::lane() == 0) *E.noise_ref = r;
}
CZ_KERNEL(k_set_opts)(EngineDev E, const uint16_t* no_act, const uint8_t* inc, const uint8_t* act, const uint8_t* hist,
                      const uint8_t* hist_given) {
  const int g = my_game();
  if (g >= E.n_games) return;
  if (E.use_history) {
    const bool given = hist && hist_given && hist_given[g];
    for (int k = czs::lane(); k < BOARD_STRIDE; k += 32)
      E.root_hist[(size_t)g * BOARD_STRIDE + k] = (given && k < NSQ) ? hist[(size_t)g * BOARD_STRIDE + k] : (uint8_t)0;
    if (czs::lane() == 0) E.root_has_hist[g] = given ? 1 : 0;
  }
  if (czs::lane() == 0) {
    int n = 0;
    if (no_act) {
      for (; n < CZ_MAX_NO_ACT; ++n) {
        const uint16_t m = no_act[(size_t)g * CZ_MAX_NO_ACT + n];
        if (m == 0xFFFF) break;
        E.no_act[(size_t)g * CZ_MAX_NO_ACT + n] = m;
      }
    }
    E.n_no_act[g] = n;
    E.increase_temp[g] = inc ? inc[g] : 0;
    E.active[g] = E.sp.retired[g] ? 0 : (act ? act[g] : 1);
  }
}

struct Carver {
  uint8_t* base; size_t off;
  template <class T> T* take(size_t count) {
    off = (off + 255) & ~(size_t)255;
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};

int next_pow2(int v) { int p = 1; while (p < v) p <<= 1; return p; }

}  // namespace

struct cz_engine {
  cz_config cfg;
  EngineDev d;
  cz_stream_t stream;
  uint8_t* ws; size_t ws_bytes;
  uint8_t* init_board_dev;
  uint8_t* opt_no_act; uint8_t* opt_inc; uint8_t* opt_act;   // device staging for cz_root_opts
  uint8_t* opt_hist; uint8_t* opt_hist_given;
  cz_pv_info* pv_dev;
  unsigned long long* stat_out;
  cz_root_info* root_info_dev;
  float* value_buf;                                         // [G*K] values of the built-in network (integrated search)
  float* legal_p;                                           // [G*K][MAX_MOVES] priors of the legal moves (integrated search)
  float* value2;                                            // eval_mirror: [2*G*K] network values of the leaves and their mirrors
  int16_t* mirror_lut;                                      // eval_mirror: [CZ_N_LABELS] cz_mirror_labels
  uint8_t* board_stage;                                     // [G][96] staging for reset / set_root
  int32_t* stat_n; uint16_t* stat_mv; int32_t* stat_cnt;    // staging for cz_get_root_stats
  int32_t* sims_stage;                                      // [G] staging for cz_set_game_sims
  int last_leaves;
  bool own_stream;                                         // e->stream was created by cz_create (caller passed the default stream)
  int ring_count;                                           // finished-game records in the device ring (as of the last cz_play_move)
  uint64_t launches;
  uint64_t total_sims;
#if !defined(CZ_EMUL)
  cznn::NnRuntime* nn;
  size_t nn_bytes;
  // the device-driven search loop as one graph: a WHILE conditional node around the iteration; [0] the production form,
  // [1] with the residual towers bracketed by the profiling stamps (captured at the first search with cz_nn_profile on)
  cudaGraphExec_t g_while[2];
  int n_ranges;                                             // 1, or 2 in arena mode (one network per range)
  volatile int32_t* h_iters;                                // mapped pinned: iterations of the last search loop (k_loop_flag)
  int32_t* d_iters;                                         // device view of h_iters
#endif
};

namespace {

size_t carve(cz_engine* e, uint8_t* base) {
  const cz_config& c = e->cfg;
  EngineDev& d = e->d;
  Carver cv{base, 0};
  const size_t G = c.n_games, K = c.leaves_per_round, N = (size_t)c.max_nodes_per_game, Ecap = (size_t)c.max_edges_per_game;
  const size_t H = (size_t)next_pow2(2 * c.max_nodes_per_game);
  d.hcap = (int)H;
  d.label_lut = cv.take<int16_t>(8100);
  d.root_board = cv.take<uint8_t>(G * BOARD_STRIDE);
  d.use_history = c.use_history ? 1 : 0;
  d.lb_stride = d.use_history ? 2 * BOARD_STRIDE : BOARD_STRIDE;
  d.root_hist = cv.take<uint8_t>(G * BOARD_STRIDE); d.root_has_hist = cv.take<int32_t>(G);
  d.root_node = cv.take<int32_t>(G); d.active = cv.take<int32_t>(G); d.tasks_left = cv.take<int32_t>(G);
  d.round_pending = cv.take<int32_t>(G); d.sims_run = cv.take<int32_t>(G); d.noise_used = cv.take<int32_t>(G);
  d.noise_epoch = cv.take<int32_t>(G);
  d.game_err = cv.take<int32_t>(G); d.no_act = cv.take<uint16_t>(G * CZ_MAX_NO_ACT); d.n_no_act = cv.take<int32_t>(G);
  d.increase_temp = cv.take<int32_t>(G);
  d.n_nodes = cv.take<int32_t>(G); d.n_edges = cv.take<int32_t>(G);
  d.node_key0 = cv.take<uint64_t>(G * N); d.node_key1 = cv.take<uint64_t>(G * N);
  d.node_sum_n = cv.take<int32_t>(G * N); d.node_edge_off = cv.take<uint32_t>(G * N); d.node_meta = cv.take<uint32_t>(G * N);
  d.node_v = cv.take<float>(G * N);
  d.hash = cv.take<uint32_t>(G * H);
  d.edge_n = cv.take<int32_t>(G * Ecap); d.edge_w = cv.take<double>(G * Ecap); d.edge_p = cv.take<float>(G * Ecap);
  d.edge_move = cv.take<uint16_t>(G * Ecap); d.edge_child = cv.take<int32_t>(G * Ecap);
  d.sim_depth = cv.take<int32_t>(G * K); d.sim_leaf_node = cv.take<int32_t>(G * K);
  d.sim_node = cv.take<int32_t>(G * K * c.max_path); d.sim_edge = cv.take<int32_t>(G * K * c.max_path);
  d.leaf_sim = cv.take<int32_t>(G * K); d.n_leaf = cv.take<int32_t>(G);
  d.leaf_board = cv.take<uint8_t>(G * K * d.lb_stride);
  d.resume_sim = cv.take<int32_t>(G * K); d.n_resume = cv.take<int32_t>(G);
  d.park_sim = cv.take<int32_t>(G * K); d.park_node = cv.take<int32_t>(G * K); d.n_park = cv.take<int32_t>(G);
  d.leaf_off = cv.take<int32_t>(G); d.totals = cv.take<int32_t>(8);
  // eval_mirror: 2*G*K rows, range h owns [2*gb*K, 2*ge*K): its n leaves, then their mirrors (k_gather)
  const size_t dense_rows = (c.eval_mirror ? 2 : 1) * G * K;
  d.leaf_dense = cv.take<uint8_t>(dense_rows * d.lb_stride);
  d.leaf_labels = cv.take<int16_t>(G * K * MAX_MOVES); d.leaf_nlab = cv.take<int32_t>(G * K);
  d.loop_iter = cv.take<int32_t>(4);
  d.noise_ref = cv.take<NoiseRef>(1);
  d.counters = cv.take<unsigned long long>(8);
  d.stat = cv.take<unsigned long long>(G * 4);
  d.gc_map = cv.take<int32_t>(G * N);
  selfplay_carve(d.sp, cv, c);
  e->init_board_dev = cv.take<uint8_t>(BOARD_STRIDE);
  e->opt_no_act = cv.take<uint8_t>(G * CZ_MAX_NO_ACT * 2); e->opt_inc = cv.take<uint8_t>(G); e->opt_act = cv.take<uint8_t>(G);
  e->opt_hist = cv.take<uint8_t>(G * BOARD_STRIDE); e->opt_hist_given = cv.take<uint8_t>(G);
  e->root_info_dev = cv.take<cz_root_info>(1);
  e->pv_dev = cv.take<cz_pv_info>(1);
  e->stat_out = cv.take<unsigned long long>(8);
  e->board_stage = cv.take<uint8_t>(G * BOARD_STRIDE);
  e->sims_stage = cv.take<int32_t>(G);
  e->stat_n = cv.take<int32_t>(G * MAX_MOVES); e->stat_mv = cv.take<uint16_t>(G * MAX_MOVES); e->stat_cnt = cv.take<int32_t>(G);
  if (c.nn_filters > 0) {
    e->value_buf = cv.take<float>(G * K);
    e->legal_p = cv.take<float>(G * K * (size_t)MAX_MOVES);
  } else {
    e->value_buf = nullptr; e->legal_p = nullptr;
  }
  if (c.eval_mirror) {
    e->value2 = cv.take<float>(2 * G * K);
    e->mirror_lut = cv.take<int16_t>(CZ_N_LABELS);
  } else {
    e->value2 = nullptr; e->mirror_lut = nullptr;
  }
  visits_carve(d.sp, cv, c);
  return cv.off + 1024;
}

int check_cfg(const cz_config* c) {
  if (!c || c->struct_bytes != (int)sizeof(cz_config)) return cz_fail(CZ_ERR_ARG, "cz_config: struct_bytes mismatch (%d vs %d)", c ? c->struct_bytes : -1, (int)sizeof(cz_config));
  if (c->n_games < 1 || c->sims_per_move < 1 || c->leaves_per_round < 1 || c->leaves_per_round > 64)
    return cz_fail(CZ_ERR_ARG, "cz_config: n_games >= 1, sims >= 1, 1 <= leaves_per_round <= 64 required");
  if (c->max_nodes_per_game < 16 || c->max_edges_per_game < 256 || c->max_path < 8)
    return cz_fail(CZ_ERR_ARG, "cz_config: pools too small");
  if (c->virtual_loss < 0 || c->max_plies < 2) return cz_fail(CZ_ERR_ARG, "cz_config: bad virtual_loss / max_plies");
  // the per-game history and record rows hold max_plies + 4 entries; the game loop writes up to 2*max_game_length (+1)
  if (c->max_game_length < 1 || c->max_plies < 2 * c->max_game_length)
    return cz_fail(CZ_ERR_ARG, "cz_config: max_game_length >= 1 and max_plies >= 2*max_game_length required (%d, %d)", c->max_game_length, c->max_plies);
  if (c->game_quota < 0 || c->playouts_lo < 0 || c->playouts_hi < c->playouts_lo)
    return cz_fail(CZ_ERR_ARG, "cz_config: bad game_quota / playouts range");
  if (c->arena && (c->n_games % 2)) return cz_fail(CZ_ERR_ARG, "cz_config: arena mode needs an even number of slots (two per game)");
  // the arena's records are scored, never trained on (evaluator.py), and its two slots per game would need a shared staging
  if (c->arena && c->record_visits) return cz_fail(CZ_ERR_ARG, "cz_config: record_visits is for self-play engines, not arena ones");
  if (c->eval_mirror != 0 && c->eval_mirror != 1) return cz_fail(CZ_ERR_ARG, "cz_config: eval_mirror must be 0 or 1");
  // the mirrored evaluation is the engine's own network run twice; an external evaluator gets the leaves as they are
  if (c->eval_mirror && c->nn_filters == 0) return cz_fail(CZ_ERR_ARG, "cz_config: eval_mirror needs the engine's own network (nn_filters > 0)");
  return 0;
}

const char kInit[] = "rkemsmekr/9/1c5c1/p1p1p1p1p/9/9/P1P1P1P1P/1C5C1/9/RKEMSMEKR";   // static_env.py:9
void init_board(uint8_t* b) {
  memset(b, 0, BOARD_STRIDE);
  int y = 9, x = 0;
  for (const char* p = kInit; *p; ++p) {
    const char ch = *p;
    if (ch == '/') { --y; x = 0; continue; }
    if (ch >= '1' && ch <= '9') { x += ch - '0'; continue; }
    uint8_t code = 0;
    switch (ch | 0x20) { case 'p': code = PC_P; break; case 'c': code = PC_C; break; case 'r': code = PC_R; break;
      case 'k': code = PC_N; break; case 'e': code = PC_E; break; case 'm': code = PC_A; break; case 's': code = PC_K; break; }
    if (ch >= 'a') code |= PC_OPP;
    b[y * 9 + x++] = code;
  }
}

// rows of the network's batch: the leaves of one search round, and with eval_mirror their mirrors too
int nn_max_batch(const cz_config* c) { return (c->eval_mirror ? 2 : 1) * c->n_games * c->leaves_per_round; }

int launch_ok(cz_engine* e, const char* what, int n = 1) {
  e->launches += n;
  const char* msg;
  const int rc = czrt_last_error(&msg);
  if (rc) return cz_fail(CZ_ERR_CUDA, "%s: %s", what, msg);
  return 0;
}

#define GAME_LAUNCH(e, kern, ...) \
  CZ_LAUNCH(kern, ((e)->cfg.n_games + kWarps - 1) / kWarps, kWarps, sizeof(TreeSmem) * kWarps, (e)->stream, __VA_ARGS__)
#define RANGE_LAUNCH(e, st, g0, g1, kern, ...) \
  CZ_LAUNCH(kern, ((g1) - (g0) + kWarps - 1) / kWarps, kWarps, sizeof(TreeSmem) * kWarps, st, __VA_ARGS__)

}  // namespace

extern "C" {

int cz_workspace_bytes(const cz_config* cfg, uint64_t* bytes) {
  if (check_cfg(cfg) || !bytes) return CZ_ERR_ARG;
  cz_engine tmp;
  tmp.cfg = *cfg;
  size_t n = carve(&tmp, nullptr);
#if !defined(CZ_EMUL)
  if (cfg->nn_filters > 0)
    n += cznn::nn_workspace_bytes(cfg->nn_filters, cfg->nn_blocks, cfg->nn_value_fc, nn_max_batch(cfg), cfg->arena ? 2 : 1,
                                  cfg->nn_policy_channels, cfg->nn_value_channels) + 4096;
#endif
  *bytes = n;
  return 0;
}

int cz_create(const cz_config* cfg, void* workspace, uint64_t workspace_bytes, void* stream, cz_engine** out) {
  if (check_cfg(cfg) || !workspace || !out) return cz_fail(CZ_ERR_ARG, "cz_create: bad argument");
  uint64_t need = 0;
  cz_workspace_bytes(cfg, &need);
  if (workspace_bytes < need) return cz_fail(CZ_ERR_ARG, "cz_create: workspace %llu < required %llu", (unsigned long long)workspace_bytes, (unsigned long long)need);
  cz_engine* e = new (std::nothrow) cz_engine();
  if (!e) return cz_fail(CZ_ERR_STATE, "cz_create: out of host memory");
  e->cfg = *cfg;
  e->stream = (cz_stream_t)stream;
  e->own_stream = false;
  e->ws = (uint8_t*)workspace; e->ws_bytes = workspace_bytes;
  e->launches = 0; e->last_leaves = 0; e->ring_count = 0; e->total_sims = 0;
  EngineDev& d = e->d;
  memset(&d, 0, sizeof(d));
  d.n_games = cfg->n_games; d.sims = cfg->sims_per_move; d.K = cfg->leaves_per_round; d.vl = cfg->virtual_loss;
  d.ncap = cfg->max_nodes_per_game; d.ecap = cfg->max_edges_per_game; d.max_path = cfg->max_path;
  d.noise_mode = cfg->noise_mode; d.max_plies = cfg->max_plies;
  d.c_puct = cfg->c_puct; d.noise_eps = cfg->noise_eps; d.alpha = cfg->dirichlet_alpha; d.tau_decay = cfg->tau_decay_rate;
  d.resign_threshold = cfg->resign_threshold; d.min_resign_turn = cfg->min_resign_turn; d.max_game_length = cfg->max_game_length;
  d.seed = cfg->seed; d.rank = cfg->rank; d.arena = cfg->arena ? 1 : 0;
  const size_t used = carve(e, e->ws);
#if !defined(CZ_EMUL)
  e->nn = nullptr; e->nn_bytes = 0;
  e->h_iters = nullptr; e->d_iters = nullptr; e->n_ranges = cfg->arena ? 2 : 1;
  e->g_while[0] = e->g_while[1] = nullptr;
  if (cudaSetDevice(cfg->device) != cudaSuccess) { delete e; return cz_fail(CZ_ERR_CUDA, "cz_create: cudaSetDevice(%d) failed", cfg->device); }
  if (!e->stream) {
    // The legacy default stream cannot be captured into a graph.  A BLOCKING stream of our own keeps the caller's ordering:
    // work the caller issues on the default stream waits for everything queued here and vice versa (implicit synchronisation
    // between the legacy default stream and blocking streams).
    if (cudaStreamCreate(&e->stream) != cudaSuccess) { delete e; return cz_fail(CZ_ERR_CUDA, "cz_create: cudaStreamCreate failed"); }
    e->own_stream = true;
  }
  if (cfg->nn_filters > 0) {
    void* hf = nullptr;
    if (cudaHostAlloc(&hf, 64, cudaHostAllocMapped) != cudaSuccess || cudaHostGetDevicePointer((void**)&e->d_iters, hf, 0) != cudaSuccess) {
      delete e; return cz_fail(CZ_ERR_CUDA, "cz_create: mapped host memory for the loop's iteration count failed");
    }
    e->h_iters = (volatile int32_t*)hf;
    memset(hf, 0, 64);
  }
#endif
  // tables + initial state
  std::vector<int16_t> lut(8100);
  cz_action_labels(nullptr, lut.data());
  czrt_copy(const_cast<int16_t*>(d.label_lut), lut.data(), 8100 * sizeof(int16_t), e->stream);
  uint8_t ib[BOARD_STRIDE];
  init_board(ib);
  czrt_copy(e->init_board_dev, ib, BOARD_STRIDE, e->stream);
  if (e->mirror_lut) {
    int16_t m[CZ_N_LABELS];
    cz_mirror_labels(m);
    czrt_copy(e->mirror_lut, m, sizeof(m), e->stream);
  }
  czrt_memset(d.counters, 0, 8 * sizeof(unsigned long long), e->stream);
  czrt_memset(d.stat, 0, (size_t)cfg->n_games * 4 * sizeof(unsigned long long), e->stream);
  czrt_sync(e->stream);
#if !defined(CZ_EMUL)
  if (cfg->nn_filters > 0) {
    const int maxb = nn_max_batch(cfg);
    e->nn_bytes = cznn::nn_workspace_bytes(cfg->nn_filters, cfg->nn_blocks, cfg->nn_value_fc, maxb, cfg->arena ? 2 : 1,
                                           cfg->nn_policy_channels, cfg->nn_value_channels);
    uint8_t* nnws = e->ws + ((used + 4095) & ~(size_t)4095);
    e->nn = cznn::nn_create(cfg->device, cfg->nn_filters, cfg->nn_blocks, cfg->nn_value_fc, maxb, nnws, e->nn_bytes, (void*)e->stream, cfg->nn_fp32_skip, cfg->arena ? 2 : 1, cfg->use_history ? 28 : 14,
                           cfg->nn_policy_channels, cfg->nn_value_channels);
    if (!e->nn) { delete e; return CZ_ERR_CUDA; }
  }
#else
  (void)used;
#endif
  *out = e;
  return cz_reset_games(e, nullptr);
}

void cz_destroy(cz_engine* e) {
  if (!e) return;
#if !defined(CZ_EMUL)
  cznn::nn_destroy(e->nn);
  if (e->h_iters) cudaFreeHost((void*)e->h_iters);
  if (e->own_stream) { cudaStreamSynchronize(e->stream); cudaStreamDestroy(e->stream); }
  for (int i = 0; i < 2; ++i)
    if (e->g_while[i]) cudaGraphExecDestroy(e->g_while[i]);
#endif
  delete e;
}

int cz_reset_games(cz_engine* e, const uint8_t* boards_host) {
  if (!e) return cz_fail(CZ_ERR_ARG, "cz_reset_games: null engine");
  const uint8_t* src = nullptr;
  if (boards_host) {
    czrt_copy(e->board_stage, boards_host, (size_t)e->cfg.n_games * BOARD_STRIDE, e->stream);
    src = e->board_stage;
  }
  GAME_LAUNCH(e, k_reset, e->d, src, (const uint8_t*)e->init_board_dev, -1);
  if (launch_ok(e, "cz_reset_games")) return CZ_ERR_CUDA;
  return czrt_sync(e->stream) ? cz_fail(CZ_ERR_CUDA, "cz_reset_games: sync failed") : 0;
}

int cz_set_root(cz_engine* e, int game, const uint8_t* board_host) {
  if (!e || game < 0 || game >= e->cfg.n_games || !board_host) return cz_fail(CZ_ERR_ARG, "cz_set_root: bad argument");
  czrt_copy(e->board_stage, board_host, BOARD_STRIDE, e->stream);
  CZ_LAUNCH(k_set_root, 1, 1, 0, e->stream, e->d, game, (const uint8_t*)e->board_stage);
  if (launch_ok(e, "cz_set_root")) return CZ_ERR_CUDA;
  return czrt_sync(e->stream) ? cz_fail(CZ_ERR_CUDA, "cz_set_root: sync failed") : 0;
}

int cz_set_roots(cz_engine* e, const uint8_t* boards_host) {
  if (!e || !boards_host) return cz_fail(CZ_ERR_ARG, "cz_set_roots: bad argument");
  czrt_copy(e->board_stage, boards_host, (size_t)e->cfg.n_games * BOARD_STRIDE, e->stream);
  GAME_LAUNCH(e, k_set_roots, e->d, (const uint8_t*)e->board_stage);
  return launch_ok(e, "cz_set_roots");
}

int cz_get_roots(cz_engine* e, uint8_t* boards_host) {
  if (!e || !boards_host) return cz_fail(CZ_ERR_ARG, "cz_get_roots: bad argument");
  czrt_copy(boards_host, e->d.root_board, (size_t)e->cfg.n_games * BOARD_STRIDE, e->stream);
  return czrt_sync(e->stream) ? cz_fail(CZ_ERR_CUDA, "cz_get_roots: device failure") : 0;
}

int cz_get_root_stats(cz_engine* e, int32_t* n_host, uint16_t* moves_host, int32_t* counts_host, int32_t* sims_run_host) {
  if (!e || !n_host || !moves_host || !counts_host) return cz_fail(CZ_ERR_ARG, "cz_get_root_stats: bad argument");
  const size_t G = e->cfg.n_games;
  GAME_LAUNCH(e, k_root_stats, e->d, e->stat_n, e->stat_mv, e->stat_cnt);
  if (launch_ok(e, "cz_get_root_stats")) return CZ_ERR_CUDA;
  czrt_copy(n_host, e->stat_n, G * MAX_MOVES * sizeof(int32_t), e->stream);
  czrt_copy(moves_host, e->stat_mv, G * MAX_MOVES * sizeof(uint16_t), e->stream);
  czrt_copy(counts_host, e->stat_cnt, G * sizeof(int32_t), e->stream);
  if (sims_run_host) czrt_copy(sims_run_host, e->d.sims_run, G * sizeof(int32_t), e->stream);
  return czrt_sync(e->stream) ? cz_fail(CZ_ERR_CUDA, "cz_get_root_stats: device failure") : 0;
}

int cz_compact(cz_engine* e) {
  if (!e) return cz_fail(CZ_ERR_ARG, "cz_compact: null engine");
  if (e->last_leaves != 0) return cz_fail(CZ_ERR_STATE, "cz_compact: a search is in flight");
  GAME_LAUNCH(e, k_compact, e->d);
  if (launch_ok(e, "cz_compact")) return CZ_ERR_CUDA;
  return czrt_sync(e->stream) ? cz_fail(CZ_ERR_CUDA, "cz_compact: device failure") : 0;
}

int cz_search_begin(cz_engine* e, const cz_root_opts* opts) {
  if (!e) return cz_fail(CZ_ERR_ARG, "cz_search_begin: null engine");
  const size_t G = e->cfg.n_games;
  const uint16_t* na = nullptr; const uint8_t* inc = nullptr; const uint8_t* act = nullptr;
  const uint8_t* hist = nullptr; const uint8_t* hist_given = nullptr;
  int sims_override = 0, raw_tasks = 0;
  NoiseRef nref{nullptr, 0};
  if (opts && opts->struct_bytes != (int)sizeof(cz_root_opts))
    return cz_fail(CZ_ERR_ARG, "cz_root_opts: struct_bytes mismatch (%d vs %d)", opts->struct_bytes, (int)sizeof(cz_root_opts));
  if (opts) {
    if (opts->no_act_host) { czrt_copy(e->opt_no_act, opts->no_act_host, G * CZ_MAX_NO_ACT * 2, e->stream); na = (const uint16_t*)e->opt_no_act; }
    if (opts->increase_temp_host) { czrt_copy(e->opt_inc, opts->increase_temp_host, G, e->stream); inc = e->opt_inc; }
    if (opts->active_host) { czrt_copy(e->opt_act, opts->active_host, G, e->stream); act = e->opt_act; }
    if (opts->root_hist_host && opts->root_hist_given_host) {
      if (!e->cfg.use_history) return cz_fail(CZ_ERR_ARG, "cz_search_begin: root history given but the engine was created without use_history");
      czrt_copy(e->opt_hist, opts->root_hist_host, G * BOARD_STRIDE, e->stream); hist = e->opt_hist;
      czrt_copy(e->opt_hist_given, opts->root_hist_given_host, G, e->stream); hist_given = e->opt_hist_given;
    }
    nref.table = opts->noise_dev; nref.stride = opts->noise_stride;
    sims_override = opts->sims_override;
    raw_tasks = opts->raw_tasks;
  }
  CZ_LAUNCH(k_set_noise, 1, 1, 0, e->stream, e->d, nref);
  if (opts) GAME_LAUNCH(e, k_set_opts, e->d, na, inc, act, hist, hist_given);   // NULL keeps the options the game loop maintains
  GAME_LAUNCH(e, k_begin, e->d, sims_override, raw_tasks);
  e->last_leaves = 0;
  return launch_ok(e, "cz_search_begin", 3);
}

int cz_set_noise_table(cz_engine* e, const double* noise_dev, int64_t noise_stride) {
  if (!e) return cz_fail(CZ_ERR_ARG, "cz_set_noise_table: null engine");
  NoiseRef nref{noise_dev, noise_stride};
  CZ_LAUNCH(k_set_noise, 1, 1, 0, e->stream, e->d, nref);
  return launch_ok(e, "cz_set_noise_table");
}

int cz_search_more(cz_engine* e, int32_t n_sims) {
  if (!e || n_sims < 0) return cz_fail(CZ_ERR_ARG, "cz_search_more: bad argument");
  if (e->last_leaves != 0) return cz_fail(CZ_ERR_STATE, "cz_search_more: %d leaves of the previous wave were not applied", e->last_leaves);
  GAME_LAUNCH(e, k_more, e->d, n_sims);
  return launch_ok(e, "cz_search_more");
}

int cz_search_wave(cz_engine* e, int32_t* n_leaves, int32_t* any_active) {
  if (!e) return cz_fail(CZ_ERR_ARG, "cz_search_wave: null engine");
  if (e->last_leaves != 0) return cz_fail(CZ_ERR_STATE, "cz_search_wave: %d leaves of the previous wave were not applied", e->last_leaves);
  const int G = e->cfg.n_games;
  RANGE_LAUNCH(e, e->stream, 0, G, k_wave, e->d, 0, G);
  CZ_LAUNCH(k_scan, 1, 1, 0, e->stream, e->d, 0, G, 0);
  RANGE_LAUNCH(e, e->stream, 0, G, k_gather, e->d, 0, G, e->d.leaf_dense, e->d.leaf_labels, e->d.leaf_nlab, (int32_t*)nullptr);
  if (launch_ok(e, "cz_search_wave", 3)) return CZ_ERR_CUDA;
  int32_t t[4];
  czrt_copy(t, e->d.totals, sizeof(t), e->stream);
  if (czrt_sync(e->stream)) return cz_fail(CZ_ERR_CUDA, "cz_search_wave: device failure");
  e->last_leaves = t[0];
  if (n_leaves) *n_leaves = t[0];
  if (any_active) *any_active = t[1] || t[0] > 0;
  return 0;
}

int cz_leaf_planes(cz_engine* e, float* planes_dev) {
  if (!e || !planes_dev) return cz_fail(CZ_ERR_ARG, "cz_leaf_planes: bad argument");
  const int n = e->last_leaves;
  if (n == 0) return 0;
  CZ_LAUNCH(k_planes_dense, (n + kWarps - 1) / kWarps, kWarps, sizeof(TreeSmem) * kWarps, e->stream,
            (const uint8_t*)e->d.leaf_dense, n, planes_dev, e->d.lb_stride);
  return launch_ok(e, "cz_leaf_planes");
}

int cz_leaf_boards(cz_engine* e, uint8_t* boards_dev) {
  if (!e || !boards_dev) return cz_fail(CZ_ERR_ARG, "cz_leaf_boards: bad argument");
  if (e->last_leaves == 0) return 0;
  return czrt_copy(boards_dev, e->d.leaf_dense, (size_t)e->last_leaves * e->d.lb_stride, e->stream) ? cz_fail(CZ_ERR_CUDA, "cz_leaf_boards: copy failed") : 0;
}

int cz_search_apply(cz_engine* e, const float* policy_dev, const float* value_dev) {
  if (!e) return cz_fail(CZ_ERR_ARG, "cz_search_apply: null engine");
  if (e->last_leaves == 0) return 0;
  if (!policy_dev || !value_dev) return cz_fail(CZ_ERR_ARG, "cz_search_apply: null evaluation");
  RANGE_LAUNCH(e, e->stream, 0, e->cfg.n_games, k_apply, e->d, 0, e->cfg.n_games, policy_dev, (const float*)nullptr, value_dev);
  e->last_leaves = 0;
  return launch_ok(e, "cz_search_apply");
}

int cz_leaf_labels(cz_engine* e, int16_t* labels_dev, int32_t* counts_dev) {
  if (!e || !labels_dev || !counts_dev) return cz_fail(CZ_ERR_ARG, "cz_leaf_labels: bad argument");
  if (e->last_leaves == 0) return 0;
  if (czrt_copy(labels_dev, e->d.leaf_labels, (size_t)e->last_leaves * MAX_MOVES * sizeof(int16_t), e->stream) ||
      czrt_copy(counts_dev, e->d.leaf_nlab, (size_t)e->last_leaves * sizeof(int32_t), e->stream))
    return cz_fail(CZ_ERR_CUDA, "cz_leaf_labels: copy failed");
  return 0;
}

int cz_search_apply_legal(cz_engine* e, const float* legal_p_dev, const float* value_dev) {
  if (!e) return cz_fail(CZ_ERR_ARG, "cz_search_apply_legal: null engine");
  if (e->last_leaves == 0) return 0;
  if (!legal_p_dev || !value_dev) return cz_fail(CZ_ERR_ARG, "cz_search_apply_legal: null evaluation");
  RANGE_LAUNCH(e, e->stream, 0, e->cfg.n_games, k_apply, e->d, 0, e->cfg.n_games, (const float*)nullptr, legal_p_dev, value_dev);
  e->last_leaves = 0;
  return launch_ok(e, "cz_search_apply_legal");
}

#if !defined(CZ_EMUL)
namespace {
// ---- device-driven search loop ------------------------------------------------------------------------------------------
// Range h = games [gb, ge) evaluated by network h (arena: player h's trees; otherwise one range = all games).  One iteration
// of a range:   apply(previous evaluation) -> wave -> scan -> gather(+labels) -> first conv | tower | heads, policy GEMM,
// legal priors.  Every launch has a fixed shape; the number of leaves is the device integer totals[4h] that k_scan writes and
// every network kernel reads, so nothing has to come back to the host between waves.
struct Range { int gb, ge; uint8_t* dense; int16_t* labels; int32_t* nlab; float* legal_p; float* value; };
Range range_of(cz_engine* e, int h) {
  const int G = e->cfg.n_games, K = e->cfg.leaves_per_round;
  const int mid = e->n_ranges == 2 ? (G + 1) / 2 : G;
  Range r;
  r.gb = h == 0 ? 0 : mid; r.ge = h == 0 ? mid : G;
  const size_t off = (size_t)r.gb * K;
  r.dense = e->d.leaf_dense + (e->cfg.eval_mirror ? 2 : 1) * off * e->d.lb_stride;
  r.labels = e->d.leaf_labels + off * MAX_MOVES; r.nlab = e->d.leaf_nlab + off;
  r.legal_p = e->legal_p + off * MAX_MOVES; r.value = e->value_buf + off;
  return r;
}
// the launches of one iteration of every range, then k_loop_flag; `cond`: the handle of the WHILE node whose body is being
// captured, null for plain launches
int enqueue_iteration(cz_engine* e, const cudaGraphConditionalHandle* cond) {
  for (int h = 0; h < e->n_ranges; ++h) {
    const Range r = range_of(e, h);
    const int n_max = (r.ge - r.gb) * e->cfg.leaves_per_round;
    RANGE_LAUNCH(e, e->stream, r.gb, r.ge, k_apply_wave, e->d, r.gb, r.ge, (const float*)r.legal_p, (const float*)r.value);
    k_scan_block<<<1, 1024, 0, e->stream>>>(e->d, r.gb, r.ge, h);
    int32_t* tot = e->d.totals + 4 * h;
    const bool mirror = e->cfg.eval_mirror != 0;
    RANGE_LAUNCH(e, e->stream, r.gb, r.ge, k_gather, e->d, r.gb, r.ge, r.dense, r.labels, r.nlab, mirror ? tot : (int32_t*)nullptr);
    const int rc = cznn::nn_forward_leaves(e->nn, e->cfg.arena ? h : 0, r.dense, n_max, tot, r.labels, r.nlab, r.legal_p, r.value,
                                           mirror ? e->mirror_lut : nullptr, mirror ? e->value2 + 2 * (size_t)r.gb * e->cfg.leaves_per_round : nullptr);
    if (rc) return rc;
  }
  CZ_LAUNCH(k_loop_flag, 1, 1, 0, e->stream, e->d, e->n_ranges, e->d_iters, cond ? (unsigned long long)*cond : 0ULL, cond ? 1 : 0);
  return 0;
}
// The whole loop as ONE graph: a WHILE conditional node whose body is one iteration of every range; k_loop_flag ends each
// iteration by setting the condition to "some range still has work".  No host involvement until the final synchronise.
// Captured with profiling as it is now (nn_profile), into g_while[profiled].
int build_while_graph(cz_engine* e, int profiled) {
  cudaGraph_t g = nullptr;
  if (cudaGraphCreate(&g, 0) != cudaSuccess) return cz_fail(CZ_ERR_CUDA, "cudaGraphCreate failed");
  cudaGraphConditionalHandle handle;
  if (cudaGraphConditionalHandleCreate(&handle, g, 1, cudaGraphCondAssignDefault) != cudaSuccess) {
    cudaGraphDestroy(g);
    return cz_fail(CZ_ERR_CUDA, "cudaGraphConditionalHandleCreate failed: %s", cudaGetErrorString(cudaGetLastError()));
  }
  cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
  np.conditional.handle = handle;
  np.conditional.type = cudaGraphCondTypeWhile;
  np.conditional.size = 1;
  cudaGraphNode_t node;
  if (cudaGraphAddNode(&node, g, nullptr, 0, &np) != cudaSuccess) {
    cudaGraphDestroy(g);
    return cz_fail(CZ_ERR_CUDA, "cudaGraphAddNode(conditional) failed: %s", cudaGetErrorString(cudaGetLastError()));
  }
  cudaGraph_t body = np.conditional.phGraph_out[0];
  int rc = 0;
  if (cudaStreamBeginCaptureToGraph(e->stream, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
    rc = cz_fail(CZ_ERR_CUDA, "cudaStreamBeginCaptureToGraph failed: %s", cudaGetErrorString(cudaGetLastError()));
  } else {
    rc = enqueue_iteration(e, &handle);
    cudaGraph_t out = nullptr;
    const cudaError_t err = cudaStreamEndCapture(e->stream, &out);
    if (!rc && err != cudaSuccess) rc = cz_fail(CZ_ERR_CUDA, "capture of the loop body failed: %s", cudaGetErrorString(err));
  }
  if (!rc && cudaGraphInstantiate(&e->g_while[profiled], g, 0) != cudaSuccess)
    rc = cz_fail(CZ_ERR_CUDA, "instantiate of the WHILE graph failed: %s", cudaGetErrorString(cudaGetLastError()));
  cudaGraphDestroy(g);
  return rc;
}
// launches per iteration of one range, for cz_launch_count (graph launches do not pass through launch_ok)
int launches_per_iteration(cz_engine* e) { return 3 + cznn::nn_launches_per_forward(e->nn); }

int search_graph_loop(cz_engine* e) {
  const int prof = cznn::nn_profiling(e->nn) ? 1 : 0;
  CZ_LAUNCH(k_loop_reset, 1, 1, 0, e->stream, e->d);
  if (!e->g_while[prof]) {
    // The first search of each form runs its first iteration as plain launches: it loads every kernel and sets their
    // attributes (neither may happen inside a stream capture) and is otherwise the same work.  The WHILE graph is captured
    // right after it and runs the rest; its body always runs once, and an iteration with no work changes nothing.
    int rc;
    if ((rc = enqueue_iteration(e, nullptr)) || (rc = build_while_graph(e, prof))) return rc;
  }
  // the whole loop is one graph launch (WHILE conditional node): the device iterates until no range has work left
  if (cudaGraphLaunch(e->g_while[prof], e->stream) != cudaSuccess)
    return cz_fail(CZ_ERR_CUDA, "cz_search: WHILE graph launch failed: %s", cudaGetErrorString(cudaGetLastError()));
  if (cudaStreamSynchronize(e->stream) != cudaSuccess) return cz_fail(CZ_ERR_CUDA, "cz_search: device failure in the loop graph");
  e->launches += (uint64_t)*e->h_iters * ((uint64_t)e->n_ranges * launches_per_iteration(e) + 1);
  const char* m;
  if (czrt_last_error(&m)) return cz_fail(CZ_ERR_CUDA, "cz_search: %s", m);
  return 0;
}
}  // namespace
#endif

int cz_search(cz_engine* e, const cz_root_opts* opts) {
#if defined(CZ_EMUL)
  (void)e; (void)opts;
  return cz_fail(CZ_ERR_UNSUPPORTED, "cz_search: the CPU emulation build has no network; use the wave/apply API");
#else
  if (!e) return cz_fail(CZ_ERR_ARG, "cz_search: null engine");
  if (!e->nn || !cznn::nn_ready(e->nn)) return cz_fail(CZ_ERR_STATE, "cz_search: network weights not set");
  int rc = cz_search_begin(e, opts);
  if (rc) return rc;
  return search_graph_loop(e);
#endif
}

int cz_search_run(cz_engine* e) {
#if defined(CZ_EMUL)
  (void)e;
  return cz_fail(CZ_ERR_UNSUPPORTED, "cz_search_run: the CPU emulation build has no network; use the wave/apply API");
#else
  if (!e) return cz_fail(CZ_ERR_ARG, "cz_search_run: null engine");
  if (!e->nn || !cznn::nn_ready(e->nn)) return cz_fail(CZ_ERR_STATE, "cz_search_run: network weights not set");
  if (e->last_leaves != 0) return cz_fail(CZ_ERR_STATE, "cz_search_run: %d leaves of a host-driven wave were not applied", e->last_leaves);
  return search_graph_loop(e);
#endif
}

int cz_get_root(cz_engine* e, int game, cz_root_info* out) {
  if (!e || !out || game < 0 || game >= e->cfg.n_games) return cz_fail(CZ_ERR_ARG, "cz_get_root: bad argument");
  CZ_LAUNCH(k_root_info, 1, 1, sizeof(TreeSmem), e->stream, e->d, game, e->root_info_dev);
  if (launch_ok(e, "cz_get_root")) return CZ_ERR_CUDA;
  czrt_copy(out, e->root_info_dev, sizeof(cz_root_info), e->stream);
  return czrt_sync(e->stream) ? cz_fail(CZ_ERR_CUDA, "cz_get_root: device failure") : 0;
}

int cz_get_pv(cz_engine* e, int game, int32_t max_len, cz_pv_info* out) {
  if (!e || !out || game < 0 || game >= e->cfg.n_games || max_len < 0 || max_len > CZ_MAX_PV)
    return cz_fail(CZ_ERR_ARG, "cz_get_pv: bad argument");
  CZ_LAUNCH(k_pv, 1, 1, sizeof(TreeSmem), e->stream, e->d, game, max_len, e->pv_dev);
  if (launch_ok(e, "cz_get_pv")) return CZ_ERR_CUDA;
  czrt_copy(out, e->pv_dev, sizeof(cz_pv_info), e->stream);
  return czrt_sync(e->stream) ? cz_fail(CZ_ERR_CUDA, "cz_get_pv: device failure") : 0;
}

int cz_get_search_stats(cz_engine* e, uint64_t* out) {
  if (!e || !out) return cz_fail(CZ_ERR_ARG, "cz_get_search_stats: bad argument");
  CZ_LAUNCH(k_stat_reduce, 1, 1, 0, e->stream, e->d, e->stat_out);
  if (launch_ok(e, "cz_get_search_stats")) return CZ_ERR_CUDA;
  unsigned long long h[6];
  czrt_copy(h, e->stat_out, sizeof(h), e->stream);
  if (czrt_sync(e->stream)) return cz_fail(CZ_ERR_CUDA, "cz_get_search_stats: device failure");
  for (int k = 0; k < 6; ++k) out[k] = h[k];
  return 0;
}

int cz_get_counters(cz_engine* e, uint64_t* out) {
  if (!e || !out) return cz_fail(CZ_ERR_ARG, "cz_get_counters: bad argument");
  unsigned long long dc[8];
  CZ_LAUNCH(k_err_reduce, 1, 1, 0, e->stream, e->d);
  czrt_copy(dc, e->d.counters, sizeof(dc), e->stream);
  if (czrt_sync(e->stream)) return cz_fail(CZ_ERR_CUDA, "cz_get_counters: device failure");
  out[0] = e->total_sims; out[1] = dc[1]; out[2] = dc[2]; out[3] = dc[3]; out[4] = dc[4];   // [1] positions, [2] waves, [3] records dropped
  out[5] = dc[5]; out[6] = dc[6]; out[7] = dc[7];
  return 0;
}

int cz_launch_count(cz_engine* e, uint64_t* n) {
  if (!e || !n) return cz_fail(CZ_ERR_ARG, "cz_launch_count: bad argument");
  uint64_t v = e->launches;
#if !defined(CZ_EMUL)
  v += cznn::nn_launches(e->nn);
#endif
  *n = v;
  return 0;
}

int cz_nn_set_weights_net(cz_engine* e, int32_t net, const cz_tensor_desc* descs, int32_t n) {
#if defined(CZ_EMUL)
  (void)e; (void)net; (void)descs; (void)n;
  return cz_fail(CZ_ERR_UNSUPPORTED, "cz_nn_set_weights: no tensor cores in the CPU emulation build");
#else
  if (!e || !descs) return cz_fail(CZ_ERR_ARG, "cz_nn_set_weights: bad argument");
  return cznn::nn_set_weights(e->nn, net, descs, n);
#endif
}

int cz_nn_set_weights(cz_engine* e, const cz_tensor_desc* descs, int32_t n) { return cz_nn_set_weights_net(e, 0, descs, n); }

int cz_nn_forward(cz_engine* e, const float* planes_dev, int32_t batch, float* policy_dev, float* value_dev) {
#if defined(CZ_EMUL)
  (void)e; (void)planes_dev; (void)batch; (void)policy_dev; (void)value_dev;
  return cz_fail(CZ_ERR_UNSUPPORTED, "cz_nn_forward: no tensor cores in the CPU emulation build");
#else
  if (!e || !planes_dev || !policy_dev || !value_dev || batch < 0) return cz_fail(CZ_ERR_ARG, "cz_nn_forward: bad argument");
  return cznn::nn_forward_planes(e->nn, 0, planes_dev, batch, policy_dev, value_dev);
#endif
}

int cz_nn_forward_boards(cz_engine* e, const uint8_t* boards_dev, int32_t batch, float* policy_dev, float* value_dev) {
#if defined(CZ_EMUL)
  (void)e; (void)boards_dev; (void)batch; (void)policy_dev; (void)value_dev;
  return cz_fail(CZ_ERR_UNSUPPORTED, "cz_nn_forward_boards: no tensor cores in the CPU emulation build");
#else
  if (!e || !boards_dev || !policy_dev || !value_dev || batch < 0) return cz_fail(CZ_ERR_ARG, "cz_nn_forward_boards: bad argument");
  return cznn::nn_forward_boards(e->nn, 0, boards_dev, batch, policy_dev, value_dev);
#endif
}

int cz_noise_sample(cz_engine* e, int game, int n_moves, int count, double* out_dev) {
  if (!e || !out_dev || count < 0 || n_moves < 1 || game < 0 || game >= e->cfg.n_games) return cz_fail(CZ_ERR_ARG, "cz_noise_sample: bad argument");
  CZ_LAUNCH(k_noise_sample, 64, 1, 0, e->stream, e->d, game, n_moves, count, out_dev);
  return launch_ok(e, "cz_noise_sample");
}

int cz_nn_profile(cz_engine* e, int enable, double* ms, uint64_t* launches, double* flops) {
#if defined(CZ_EMUL)
  (void)e; (void)enable; (void)ms; (void)launches; (void)flops;
  return cz_fail(CZ_ERR_UNSUPPORTED, "cz_nn_profile: no network in the CPU emulation build");
#else
  if (!e || !e->nn) return cz_fail(CZ_ERR_STATE, "cz_nn_profile: engine has no network");
  cznn::nn_profile(e->nn, enable != 0);
  return cznn::nn_profile_read(e->nn, ms, launches, flops);           // synchronises the stream
#endif
}

int cz_nn_read_buffer(cz_engine* e, int32_t which, int32_t n, void* dst_dev, int64_t dst_bytes, int64_t* row_bytes) {
#if defined(CZ_EMUL)
  (void)e; (void)which; (void)n; (void)dst_dev; (void)dst_bytes; (void)row_bytes;
  return cz_fail(CZ_ERR_UNSUPPORTED, "cz_nn_read_buffer: no network in the CPU emulation build");
#else
  if (!e || !e->nn) return cz_fail(CZ_ERR_STATE, "cz_nn_read_buffer: engine has no network");
  long long rb = 0;
  const int rc = cznn::nn_read_buffer(e->nn, which, n, dst_dev, (long long)dst_bytes, &rb);
  if (row_bytes) *row_bytes = rb;
  return rc;
#endif
}

}  // extern "C"

#include "cz_selfplay_api.inc"
