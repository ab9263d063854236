// cz_tree.cuh — PUCT search over per-game transposition tables, warp-per-game device code.
//
// Replaces agent/player.py of the reference: VisitState/ActionState (:17-33) become SoA node/edge
// pools keyed by a 128-bit position key (the reference keys a dict by state string, :49,211);
// MCTS_search (:198-260), select_action_q_and_u (:262-320), expand (:211-221), update_tree (:340-373)
// and the round scheduling of action() (:167-179) become the wave / apply kernels below, following the
// canonical schedule of SURVEY.md Appendix C (one FIFO worker; network replies when the queue is dry).
//
// Arithmetic contract (numpy-2 semantics of the reference expressions, see oracle/player.py):
//   priors P are float32; all_p is a sequential float32 sum in legal-move order; W, Q, U, the score
//   and sqrt(sum_n+1) are float64; c_puct*P and (1-eps)*P are float32 products; compiled with
//   -fmad=false / -ffp-contract=off so no product-sum is fused.
#pragma once
#include "cz_env.cuh"

namespace cz {

enum { CHILD_UNKNOWN = -1, CHILD_TERM_BASE = -2 };        // child <= -2: terminal, v = (-2 - child) - 1
enum { NODE_WAITING = 1u << 8 };
enum { GAME_ERR_PATH = 1, GAME_ERR_POOL = 2, GAME_ERR_NOISE = 4, GAME_ERR_NOMOVE = 8 };

struct RecordHdr { int32_t n_plies, value_red, game_index, flags; };
struct NoiseRef { const double* table; long long stride; };

// per-game state of the on-device game loop (cz_selfplay.cuh)
struct SelfplayDev {
  int32_t* turns;          // [G] plies played in the current game
  int32_t* no_eat;         // [G] consecutive non-capturing plies
  int32_t* enable_resign;  // [G]
  int32_t* games_started;  // [G] games begun in this slot (RNG stream + game index)
  int32_t* sims_game;      // [G] simulations per move of the game in this slot (evaluator.py:153-154), 0 = EngineDev::sims
  int32_t* retired;        // [G] 1 = the slot reached cz_config.game_quota and plays no further game
  uint64_t* hist_k0;       // [G][hist_stride] keys of the states s_0..s_turns
  uint64_t* hist_k1;
  uint16_t* hist_move;     // [G][hist_stride] actions a_0..a_{turns-1}
  RecordHdr* rec_hdr;      // [rec_cap]
  uint16_t* rec_moves;     // [rec_cap][hist_stride]
  int32_t* rec_count;      // [1] records in the ring
  int32_t* finished;       // [1] games finished by the last cz_play_move
  // cz_config.record_visits: every ply's root visit counts (calc_policy's N(s,a), player.py:375-406).  Staging per game
  // (ascending label order within a ply), copied at game end into a pair heap beside the ring (cz_record_visits_layout)
  uint16_t* vis_lab;       // [G][hist_stride * MAX_MOVES] staged labels of the game in the slot
  uint32_t* vis_n;         // [G][hist_stride * MAX_MOVES] staged N
  uint8_t* vis_ply;        // [G][hist_stride] pairs per ply (0 for an appended final king capture)
  int32_t* vis_cursor;     // [G] pairs staged so far
  unsigned long long* vis_used;  // [1] pairs claimed in the heap (bump allocator)
  int64_t* rec_vis_off;    // [rec_cap] first heap pair of the record
  uint8_t* rec_vis_cnt;    // [rec_cap][hist_stride] pairs per ply of the record
  uint32_t* vis_heap;      // [rec_cap * hist_stride * MAX_MOVES][2] (label, N)
  int32_t record_visits;
  int32_t rec_cap, hist_stride;
  int32_t game_quota, playouts_lo, playouts_hi;
  double enable_resign_rate;
};

struct EngineDev {
  // ---- configuration
  int n_games, sims, K, vl, ncap, ecap, hcap, max_path, noise_mode, max_plies;
  double c_puct, noise_eps, alpha, tau_decay, resign_threshold;
  int min_resign_turn, max_game_length;
  uint64_t seed; int rank;
  int arena;                     // 1: slots g and g + G/2 are the two players' trees of one game (worker/evaluator.py)
  int use_history;               // 28 input planes (static_env.py:158-194): every leaf carries a second board
  int lb_stride;                 // bytes per leaf record: BOARD_STRIDE, or 2*BOARD_STRIDE (board, history board) with use_history
  // ---- tables
  const int16_t* label_lut;      // [8100]
  // ---- per game: root + search bookkeeping
  uint8_t* root_board;           // [G][96]
  uint8_t* root_hist;            // [G][96] use_history: hist[-5] of action()'s `hist` argument (all empty = zero planes)
  int32_t* root_has_hist;        // [G]     use_history: action() was given a non-empty `hist`
  int32_t* root_node;            // [G]
  int32_t* active;               // [G]
  int32_t* tasks_left;           // [G]
  int32_t* round_pending;        // [G]
  int32_t* sims_run;             // [G]
  int32_t* noise_used;           // [G]
  int32_t* noise_epoch;          // [G] searches opened on this slot since the last reset: part of the Philox counter of the root
                                 //     noise, so that every move of every game draws from its own stream
  int32_t* game_err;             // [G]
  uint16_t* no_act;              // [G][16]
  int32_t* n_no_act;             // [G]
  int32_t* increase_temp;        // [G]
  // Root-noise table of the open search (noise_mode 0).  EngineDev travels BY VALUE into kernel launches that may be frozen
  // inside a captured CUDA graph, so everything that changes per search lives behind a device pointer:
  NoiseRef* noise_ref;           // [1] {table, stride}, rewritten by cz_search_begin / cz_set_noise_table
  // ---- tree pools (per game segments)
  int32_t* n_nodes;              // [G]
  int32_t* n_edges;              // [G]
  uint64_t* node_key0;           // [G*ncap]
  uint64_t* node_key1;
  int32_t* node_sum_n;
  uint32_t* node_edge_off;
  uint32_t* node_meta;           // nedge | flags
  float* node_v;                 // network value of the node's position (player.py:349-350 `debug[state]`, read by the PV line)
  uint32_t* hash;                // [G*hcap] 0 = empty else node+1
  int32_t* edge_n;               // [G*ecap]
  double* edge_w;
  float* edge_p;
  uint16_t* edge_move;
  int32_t* edge_child;
  // ---- simulations of the current round
  int32_t* sim_depth;            // [G*K]
  int32_t* sim_leaf_node;        // [G*K]
  int32_t* sim_node;             // [G*K*max_path]
  int32_t* sim_edge;             // [G*K*max_path]
  int32_t* leaf_sim;             // [G*K]
  int32_t* n_leaf;               // [G]
  uint8_t* leaf_board;           // [G*K][lb_stride]
  int32_t* resume_sim;           // [G*K]
  int32_t* n_resume;             // [G]
  int32_t* park_sim;             // [G*K]
  int32_t* park_node;            // [G*K]
  int32_t* n_park;               // [G]
  int32_t* leaf_off;             // [G]
  int32_t* totals;               // [4]: total leaves, any active, -, -
  uint8_t* leaf_dense;           // [G*K][lb_stride] leaves of all games, dense
  int16_t* leaf_labels;          // [G*K][MAX_MOVES] dense: action label of every legal move of the leaf (-1 = none)
  int32_t* leaf_nlab;            // [G*K] dense: legal moves of the leaf
  int32_t* loop_iter;            // [1] iterations of the device-driven search loop finished (k_loop_flag)
  unsigned long long* counters;  // [8]
  unsigned long long* stat;      // [G][4] since cz_create: simulations backed up, sum of their path lengths, simulations
                                 //        that ended without the network (terminal / repetition / error), nodes created
  int32_t* gc_map;               // [G*ncap] scratch of game_compact: old node -> new node + 1 (0 = dropped)
  SelfplayDev sp;
};

struct TreeSmem {                // per warp
  uint8_t board[BOARD_STRIDE];
  move_t list[MAX_MOVES];
  float pr[MAX_MOVES];
  EnvScratch sc;
  int32_t imm_sim[64];
  double imm_val[64];
};

// ------------------------------------------------------------------ counter-based RNG (noise_mode 1)
CZ_HD void philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t* out) {
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
struct Rng {                     // a private stream: key = (seed, rank), counter = (game, purpose, index, block)
  uint32_t k0, k1, c0, c1, c2, blk, buf[4]; int have;
  CZ_DM void init(uint64_t seed, int rank, uint32_t game, uint32_t purpose, uint32_t index) {
    k0 = (uint32_t)seed ^ (uint32_t)(rank * 0x632BE5ABu); k1 = (uint32_t)(seed >> 32) + 0x1234567u * (uint32_t)rank;
    c0 = game; c1 = purpose; c2 = index; blk = 0; have = 0;
  }
  CZ_DM uint32_t next() {
    if (!have) { philox4x32(c0, c1, c2, blk++, k0, k1, buf); have = 4; }
    return buf[--have];
  }
  CZ_DM double uniform() {       // (0,1)
    const uint64_t a = next(), b = next();
    return ((double)(((a << 32) | b) >> 11) + 0.5) * (1.0 / 9007199254740992.0);
  }
  // The root-noise sampler below works in single precision with the SFU transcendentals: the draws only have to be
  // Beta(alpha, (L-1) alpha) distributed (tests/test_noise.py), and in fp64 (log / cos / pow slow paths) they were 35 %
  // of all instructions k_wave executed (ncu source view, profiles/).  uniform() above stays fp64: the move / resign /
  // store lotteries are restated bit for bit by oracle/selfplay.py.
  CZ_DM float uniform_f() {      // (0,1), 24 bits, never 0 or 1
    return ((float)(next() >> 8) + 0.5f) * (1.0f / 16777216.0f);
  }
  CZ_DM float normal_f() {
    const float u1 = uniform_f(), u2 = uniform_f();
    return czs::fsqrt(-2.0f * czs::flog(u1)) * czs::fcos(6.2831853f * u2);
  }
  CZ_DM float gamma_f(float a) { // Marsaglia-Tsang, with the a < 1 boost
    float boost = 1.0f;
    if (a < 1.0f) { boost = czs::fpow(uniform_f(), 1.0f / a); a += 1.0f; }
    const float d = a - 1.0f / 3.0f, c = 1.0f / czs::fsqrt(9.0f * d);
    for (int it = 0; it < 64; ++it) {
      const float x = normal_f();
      float v = 1.0f + c * x;
      if (v <= 0.0f) continue;
      v = v * v * v;
      const float u = uniform_f();
      if (czs::flog(u) < 0.5f * x * x + d - d * v + d * czs::flog(v)) return d * v * boost;
    }
    return d * boost;
  }
};
// first component of Dirichlet(alpha * 1_n): Gamma(alpha) / (Gamma(alpha) + Gamma((n-1) alpha))
CZ_D double dirichlet_first(const EngineDev& E, int game, uint32_t index, int n) {
  Rng r; r.init(E.seed, E.rank, (uint32_t)game, 1u | ((uint32_t)E.noise_epoch[game] << 8), index);
  const float g1 = r.gamma_f((float)E.alpha);
  if (n <= 1) return 1.0;
  const float g2 = r.gamma_f((float)E.alpha * (float)(n - 1));
  const float s = g1 + g2;
  return s > 0.0f ? (double)(g1 / s) : 0.0;
}

// ------------------------------------------------------------------ transposition table
// Linear probing, 32 slots per step: lane i looks at slot s + i (one round trip of hash + key loads for the whole probe
// sequence instead of one dependent round trip per slot).  The key, if stored, sits before the first empty slot.
CZ_D int tt_lookup(const EngineDev& E, int g, uint64_t k0, uint64_t k1) {
  const uint32_t mask = (uint32_t)E.hcap - 1;
  const uint32_t* h = E.hash + (size_t)g * E.hcap;
  const uint32_t s0 = (uint32_t)k0 & mask;
  for (int base = 0; base < E.hcap; base += 32) {
    const uint32_t v = h[(s0 + (uint32_t)(base + czs::lane())) & mask];
    bool match = false;
    if (v != 0) {
      const size_t ni = (size_t)g * E.ncap + (v - 1);
      match = E.node_key0[ni] == k0 && E.node_key1[ni] == k1;
    }
    const unsigned m_empty = czs::ballot(v == 0), m_match = czs::ballot(match);
    const unsigned before = m_empty ? ((1u << (czs::ffs(m_empty) - 1)) - 1u) : 0xffffffffu;   // lanes ahead of the first empty slot
    if (m_match & before) return (int)czs::shfl(v, czs::ffs(m_match & before) - 1) - 1;
    if (m_empty) return -1;
  }
  return -1;
}
CZ_D void tt_insert(const EngineDev& E, int g, uint64_t k0, int node) {
  const uint32_t mask = (uint32_t)E.hcap - 1;
  uint32_t* h = E.hash + (size_t)g * E.hcap;
  const uint32_t s0 = (uint32_t)k0 & mask;
  for (int base = 0; base < E.hcap; base += 32) {
    const uint32_t slot = (s0 + (uint32_t)(base + czs::lane())) & mask;
    const unsigned m_empty = czs::ballot(h[slot] == 0);
    if (m_empty) {
      if (czs::lane() == czs::ffs(m_empty) - 1) h[slot] = (uint32_t)node + 1;      // the first empty slot of the probe sequence
      break;
    }
  }
  czs::syncwarp();
}

// New node for the position on `board` with the ordered move list (expand, player.py:211-221).
// Returns the node index or -1 when a pool is exhausted.
CZ_D int node_create(const EngineDev& E, int g, uint64_t k0, uint64_t k1, const move_t* list, int L) {
  const int nn = E.n_nodes[g], ne = E.n_edges[g];
  czs::syncwarp();                                   // every lane has read the counters before lane 0 bumps them
  if (nn + 1 > E.ncap || ne + L > E.ecap) return -1;
  const size_t ni = (size_t)g * E.ncap + nn;
  const size_t eo = (size_t)g * E.ecap + ne;
  for (int i = czs::lane(); i < L; i += 32) {
    E.edge_n[eo + i] = 0; E.edge_w[eo + i] = 0.0; E.edge_p[eo + i] = 0.f;
    E.edge_move[eo + i] = list[i]; E.edge_child[eo + i] = CHILD_UNKNOWN;
  }
  if (czs::lane() == 0) {
    E.node_key0[ni] = k0; E.node_key1[ni] = k1;
    E.node_sum_n[ni] = 1;
    E.node_edge_off[ni] = (uint32_t)ne;
    E.node_meta[ni] = (uint32_t)L | NODE_WAITING;
    E.n_nodes[g] = nn + 1; E.n_edges[g] = ne + L;
    E.stat[(size_t)g * 4 + 3] += 1;
  }
  czs::syncwarp();
  tt_insert(E, g, k0, nn);
  return nn;
}

// ------------------------------------------------------------------ select (player.py:262-320)
// Returns the local edge index, or -1 if the node has no selectable edge.
CZ_D int select_edge(const EngineDev& E, int g, int node, bool is_root) {
  const size_t ni = (size_t)g * E.ncap + node;
  const int L = (int)(E.node_meta[ni] & 0xff);
  const size_t eo = (size_t)g * E.ecap + E.node_edge_off[ni];
  const double xx = czs::dsqrt((double)(E.node_sum_n[ni] + 1));
  const float cpf = (float)E.c_puct, omef = (float)(1.0 - E.noise_eps);
  const int nna = is_root ? E.n_no_act[g] : 0;
  const uint16_t* na = E.no_act + (size_t)g * CZ_MAX_NO_ACT;
  const int cursor = E.noise_used[g];
  const NoiseRef nref = (is_root && E.noise_mode == 0) ? *E.noise_ref : NoiseRef{nullptr, 0};
  double best_s = -99999999.0; int best_i = -1;
  int first_big = 0x7fffffff;
  int seen = 0;                                   // non-skipped edges before this chunk
  for (int base = 0; base < L; base += 32) {
    const int i = base + czs::lane();
    const bool valid = i < L;
    int n = 0; double w = 0.0; float p = 0.f; bool skip = !valid;
    if (valid) {
      n = E.edge_n[eo + i]; w = E.edge_w[eo + i]; p = E.edge_p[eo + i];
      if (nna) { const uint16_t m = E.edge_move[eo + i]; for (int k = 0; k < nna; ++k) skip = skip || na[k] == m; }
    }
    const unsigned live = czs::ballot(!skip);
    const int rank = seen + czs::popc(live & ((1u << czs::lane()) - 1u));
    double score = -1e300; bool big = false;
    if (!skip) {
      const double q = n != 0 ? w / (double)n : 0.0;
      double cp_p;
      if (is_root) {
        double nz;
        if (E.noise_mode == 0) {
          nz = (nref.table && (long long)cursor + rank < nref.stride)
                   ? nref.table[(size_t)g * nref.stride + cursor + rank] : 0.0;
        } else if (E.noise_eps == 0.0) {
          nz = 0.0;                                 // eps * nz adds +0.0 whatever the draw: the cursor advances, nothing is sampled
        } else {
          nz = dirichlet_first(E, g, (uint32_t)(cursor + rank), L);
        }
        const double pmix = (double)(omef * p) + E.noise_eps * nz;
        cp_p = E.c_puct * pmix;
      } else {
        cp_p = (double)(cpf * p);
      }
      score = q + cp_p * xx / (double)(1 + n);
      big = q > (1.0 - 1e-7);
    }
    const unsigned bigm = czs::ballot(big);
    if (bigm && first_big == 0x7fffffff) first_big = base + czs::ffs(bigm) - 1;
    // warp arg-max, later index wins ties (the reference's `>=`)
    double s = score; int idx = skip ? -1 : i;
    for (int m = 16; m; m >>= 1) {
      const double os = czs::shfl_xor(s, m); const int oi = czs::shfl_xor(idx, m);
      if (oi >= 0 && (idx < 0 || os > s || (os == s && oi > idx))) { s = os; idx = oi; }
    }
    if (idx >= 0 && s >= best_s) { best_s = s; best_i = idx; }
    if (first_big != 0x7fffffff) {                 // `break` at the first q > 1-1e-7
      const int upto = first_big - base;           // lanes 0..upto of this chunk drew noise
      seen += czs::popc(live & (upto >= 31 ? 0xffffffffu : ((2u << upto) - 1u)));
      break;
    }
    seen += czs::popc(live);
  }
  if (is_root) {
    if (E.noise_mode == 0 && nref.table && (long long)cursor + seen > nref.stride && czs::lane() == 0)
      E.game_err[g] |= GAME_ERR_NOISE;
    if (czs::lane() == 0) E.noise_used[g] = cursor + seen;
    czs::syncwarp();
  }
  return first_big != 0x7fffffff ? first_big : best_i;
}

// ------------------------------------------------------------------ backup (update_tree, player.py:355-366)
// One lane per path level: the edges of a path are distinct (a repeated node ends the simulation before it is selected from
// again), so the read-modify-writes are independent and cost one memory round trip instead of one per level.  The value
// alternates in sign from the leaf upwards (v = -v before every level, :357-359); negation is exact, so every edge receives
// bit for bit what the sequential loop would add.
CZ_D void backup(const EngineDev& E, int g, int sim, double v) {
  const size_t so = ((size_t)g * E.K + sim) * E.max_path;
  const int depth = E.sim_depth[(size_t)g * E.K + sim];
  const double vl = (double)E.vl;
  for (int base = 0; base < depth; base += 32) {
    const int l = base + czs::lane();
    if (l < depth) {
      const double vs = ((depth - l) & 1) ? -v : v;
      const size_t e = (size_t)g * E.ecap + E.sim_edge[so + l];
      E.edge_n[e] += 1 - E.vl;
      E.edge_w[e] = E.edge_w[e] + (vs + vl);
    }
  }
  if (czs::lane() == 0) { E.stat[(size_t)g * 4 + 0] += 1; E.stat[(size_t)g * 4 + 1] += (unsigned long long)depth; }
  czs::syncwarp();
}

// ------------------------------------------------------------------ one simulation descent (MCTS_search)
// Outcome codes returned to the wave loop.
enum { OUT_LEAF = 0, OUT_IMMEDIATE = 1, OUT_PARKED = 2 };

CZ_D int descend(const EngineDev& E, int g, int sim, bool fresh, TreeSmem* sm, double* imm_value) {
  const size_t si = (size_t)g * E.K + sim;
  const size_t so = si * E.max_path;
  int depth, cur;
  copy_board(E.root_board + (size_t)g * BOARD_STRIDE, sm->board);
  if (fresh) {
    depth = 0;
    cur = E.root_node[g] >= 0 ? E.root_node[g] : CHILD_UNKNOWN;
  } else {
    depth = E.sim_depth[si];
    for (int l = 0; l < depth; ++l)
      step_flip(sm->board, E.edge_move[(size_t)g * E.ecap + E.sim_edge[so + l]], sm->board);
    cur = E.sim_leaf_node[si];                       // the node it parked on
  }
  int parent_edge = depth > 0 ? E.sim_edge[so + depth - 1] : -1;
  for (;;) {
    if (cur == CHILD_UNKNOWN) {
      uint64_t k0, k1;
      board_key(sm->board, &k0, &k1);
      int found = tt_lookup(E, g, k0, k1);
      if (found < 0) {
        int nm;
        const DoneResult dr = done_eval(sm->board, sm->list, &nm, false, sm->sc.b0, sm->sc.l0);
        if (dr.over) {
          if (parent_edge >= 0 && czs::lane() == 0) E.edge_child[(size_t)g * E.ecap + parent_edge] = CHILD_TERM_BASE - (dr.v + 1);
          if (czs::lane() == 0) E.sim_depth[si] = depth;
          czs::syncwarp();
          *imm_value = 2.0 * (double)dr.v;          // v * 2 (player.py:206)
          return OUT_IMMEDIATE;
        }
        const int node = node_create(E, g, k0, k1, sm->list, nm);
        if (node < 0) {                              // pool exhausted: count it and finish the sim as a draw
          if (czs::lane() == 0) { E.game_err[g] |= GAME_ERR_POOL; E.sim_depth[si] = depth; }
          czs::syncwarp();
          *imm_value = 0.0;
          return OUT_IMMEDIATE;
        }
        const int j = E.n_leaf[g];                   // leaf slot of this game (every lane reads before lane 0 bumps it)
        czs::syncwarp();
        if (czs::lane() == 0) {
          if (parent_edge >= 0) E.edge_child[(size_t)g * E.ecap + parent_edge] = node;
          if (depth == 0) E.root_node[g] = node;
          E.sim_depth[si] = depth;
          E.sim_leaf_node[si] = node;
          E.leaf_sim[(size_t)g * E.K + j] = sim;
          E.n_leaf[g] = j + 1;
        }
        uint8_t* lb = E.leaf_board + ((size_t)g * E.K + j) * E.lb_stride;
        for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) lb[k] = k < NSQ ? sm->board[k] : (uint8_t)0;
        if (E.use_history) {
          // expand_and_evaluate (player.py:322-334): planes 14-27 come from history[-5].  A descent that started at the
          // root of an action() call that was given `hist` uses that list for every leaf it expands (is_root_node is
          // never cleared, :198-221); otherwise the path: the position two plies above the leaf, none for depth < 2.
          const uint8_t* hsrc = nullptr;
          if (fresh && E.root_has_hist[g]) hsrc = E.root_hist + (size_t)g * BOARD_STRIDE;
          else if (depth >= 2) {
            copy_board(E.root_board + (size_t)g * BOARD_STRIDE, sm->sc.b0);
            for (int l = 0; l < depth - 2; ++l)
              step_flip(sm->sc.b0, E.edge_move[(size_t)g * E.ecap + E.sim_edge[so + l]], sm->sc.b0);
            hsrc = sm->sc.b0;
          }
          for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) lb[BOARD_STRIDE + k] = (hsrc && k < NSQ) ? hsrc[k] : (uint8_t)0;
        }
        czs::syncwarp();
        return OUT_LEAF;
      }
      cur = found;
      if (parent_edge >= 0 && czs::lane() == 0) E.edge_child[(size_t)g * E.ecap + parent_edge] = cur;
    }
    if (cur <= CHILD_TERM_BASE) {                    // cached terminal child
      if (czs::lane() == 0) E.sim_depth[si] = depth;
      czs::syncwarp();
      *imm_value = 2.0 * (double)((CHILD_TERM_BASE - cur) - 1);
      return OUT_IMMEDIATE;
    }
    // ---- the state is in the tree
    // loop check: `state in history[:-1]` (player.py:223-234), first earlier occurrence decides
    int rep = 0x7fffffff;
    for (int l = czs::lane(); l < depth; l += 32)
      if (E.sim_node[so + l] == cur && l < rep) rep = l;
    for (int m = 16; m; m >>= 1) { const int o = czs::shfl_xor(rep, m); rep = o < rep ? o : rep; }
    if (rep != 0x7fffffff) {
      const move_t mv = E.edge_move[(size_t)g * E.ecap + E.sim_edge[so + rep]];
      double v;
      if (will_check_or_catch(sm->board, mv, &sm->sc)) v = -1.0;
      else if (be_catched(sm->board, mv, &sm->sc)) v = 1.0;
      else v = 0.0;
      if (czs::lane() == 0) E.sim_depth[si] = depth;
      czs::syncwarp();
      *imm_value = v;
      return OUT_IMMEDIATE;
    }
    const size_t ni = (size_t)g * E.ncap + cur;
    if (E.node_meta[ni] & NODE_WAITING) {            // park until the evaluation arrives (:238-241)
      if (czs::lane() == 0) {
        E.sim_depth[si] = depth;
        E.sim_leaf_node[si] = cur;
        const int k = E.n_park[g];
        E.park_sim[(size_t)g * E.K + k] = sim;
        E.park_node[(size_t)g * E.K + k] = cur;
        E.n_park[g] = k + 1;
      }
      czs::syncwarp();
      return OUT_PARKED;
    }
    const int e = select_edge(E, g, cur, cur == E.root_node[g]);
    if (e < 0) {                                     // no playable edge (reference would fail here)
      if (czs::lane() == 0) { E.game_err[g] |= GAME_ERR_NOMOVE; E.sim_depth[si] = depth; }
      czs::syncwarp();
      *imm_value = 0.0;
      return OUT_IMMEDIATE;
    }
    if (depth >= E.max_path) {
      if (czs::lane() == 0) { E.game_err[g] |= GAME_ERR_PATH; E.sim_depth[si] = depth; }
      czs::syncwarp();
      *imm_value = 0.0;
      return OUT_IMMEDIATE;
    }
    const int eabs = (int)E.node_edge_off[ni] + e;
    const size_t ei = (size_t)g * E.ecap + eabs;
    if (czs::lane() == 0) {                          // virtual loss (:245-252)
      E.node_sum_n[ni] += 1;
      E.edge_n[ei] += E.vl;
      E.edge_w[ei] = E.edge_w[ei] - (double)E.vl;
      E.sim_node[so + depth] = cur;
      E.sim_edge[so + depth] = eabs;
    }
    czs::syncwarp();
    ++depth;
    parent_edge = eabs;
    step_flip(sm->board, E.edge_move[ei], sm->board);
    cur = E.edge_child[ei];
  }
}

// ------------------------------------------------------------------ wave: run queued simulations of one game
CZ_D void game_wave(const EngineDev& E, int g, TreeSmem* sm) {
  if (!E.active[g]) { if (czs::lane() == 0) E.n_leaf[g] = 0; return; }
  if (czs::lane() == 0) E.n_leaf[g] = 0;
  czs::syncwarp();
  for (;;) {
    int n_queue; bool fresh;
    if (E.round_pending[g] == 0) {
      const int left = E.tasks_left[g];
      if (left <= 0) return;                         // this move's search is complete
      n_queue = left < E.K ? left : E.K;
      fresh = true;
      czs::syncwarp();
      if (czs::lane() == 0) { E.tasks_left[g] = left - n_queue; E.round_pending[g] = n_queue; E.n_park[g] = 0; E.n_resume[g] = 0; }
      czs::syncwarp();
    } else {
      n_queue = E.n_resume[g];
      fresh = false;
      if (n_queue == 0) return;                      // waiting for evaluations only
    }
    int n_imm = 0;
    for (int qi = 0; qi < n_queue; ++qi) {
      const int sim = fresh ? qi : E.resume_sim[(size_t)g * E.K + qi];
      double v = 0.0;
      const int out = descend(E, g, sim, fresh, sm, &v);
      if (out == OUT_IMMEDIATE) {
        if (czs::lane() == 0) { sm->imm_sim[n_imm] = sim; sm->imm_val[n_imm] = v; }
        ++n_imm;
      }
    }
    czs::syncwarp();
    if (!fresh && czs::lane() == 0) E.n_resume[g] = 0;
    // terminal / repetition results are backed up after every queued descent, in order
    for (int i = 0; i < n_imm; ++i) backup(E, g, sm->imm_sim[i], sm->imm_val[i]);
    czs::syncwarp();
    if (czs::lane() == 0) {
      E.round_pending[g] -= n_imm;
      E.sims_run[g] += n_imm;
      E.stat[(size_t)g * 4 + 2] += (unsigned long long)n_imm;
    }
    czs::syncwarp();
    if (E.n_leaf[g] > 0 || E.round_pending[g] > 0) return;   // evaluations outstanding
    // the whole round finished without the network: open the barrier and start the next round
  }
}

// ------------------------------------------------------------------ apply: attach evaluations, back up, resume
// policy: [n][2086] softmax vectors (external evaluators: the reference's wire format), or — legal_p != null — the same
// probabilities already gathered at the leaf's legal-move labels, [n][MAX_MOVES] (integrated search: the 2086-vector is
// never materialised).  Everything after the gather is identical.
CZ_D void game_apply(const EngineDev& E, int g, const float* policy, const float* legal_p, const float* value, TreeSmem* sm) {
  const int nl = E.n_leaf[g];
  if (nl == 0) return;
  const int off = E.leaf_off[g];
  int n_res = 0;
  for (int j = 0; j < nl; ++j) {
    const int sim = E.leaf_sim[(size_t)g * E.K + j];
    const int node = E.sim_leaf_node[(size_t)g * E.K + sim];
    const size_t ni = (size_t)g * E.ncap + node;
    const int L = (int)(E.node_meta[ni] & 0xff);
    const size_t eo = (size_t)g * E.ecap + E.node_edge_off[ni];
    // priors of the legal moves, renormalised (player.py:272-284): float32, sequential sum
    if (legal_p) {
      const float* lrow = legal_p + (size_t)(off + j) * MAX_MOVES;
      for (int i = czs::lane(); i < L; i += 32) sm->pr[i] = lrow[i];
    } else {
      const float* prow = policy + (size_t)(off + j) * N_LABELS;
      for (int i = czs::lane(); i < L; i += 32) {
        const move_t m = E.edge_move[eo + i];
        const int lab = E.label_lut[mv_from(m) * 90 + mv_to(m)];
        sm->pr[i] = lab >= 0 ? prow[lab] : 0.f;
      }
    }
    czs::syncwarp();
    float all_p = 0.f;
    if (czs::lane() == 0) { for (int i = 0; i < L; ++i) all_p = all_p + sm->pr[i]; if (all_p == 0.f) all_p = 1.f; }
    all_p = czs::shfl(all_p, 0);
    for (int i = czs::lane(); i < L; i += 32) E.edge_p[eo + i] = sm->pr[i] / all_p;
    if (czs::lane() == 0) { E.node_meta[ni] &= ~(uint32_t)NODE_WAITING; E.node_v[ni] = value[off + j]; }
    czs::syncwarp();
    // simulations parked on this node re-enter the queue in park order (:351-353)
    const int np = E.n_park[g];
    if (czs::lane() == 0) {
      for (int k = 0; k < np; ++k)
        if (E.park_node[(size_t)g * E.K + k] == node) {
          E.resume_sim[(size_t)g * E.K + n_res++] = E.park_sim[(size_t)g * E.K + k];
          E.park_node[(size_t)g * E.K + k] = -1;
        }
    }
    n_res = czs::shfl(n_res, 0);
    backup(E, g, sim, (double)value[off + j]);
  }
  if (czs::lane() == 0) {
    int w = 0;                                       // drop resolved park entries
    const int np = E.n_park[g];
    for (int k = 0; k < np; ++k)
      if (E.park_node[(size_t)g * E.K + k] >= 0) {
        E.park_node[(size_t)g * E.K + w] = E.park_node[(size_t)g * E.K + k];
        E.park_sim[(size_t)g * E.K + w] = E.park_sim[(size_t)g * E.K + k];
        ++w;
      }
    E.n_park[g] = w;
    E.n_resume[g] = n_res;
    E.round_pending[g] -= nl;
    E.sims_run[g] += nl;
    E.n_leaf[g] = 0;
  }
  czs::syncwarp();
}

// ------------------------------------------------------------------ pool compaction
// Keep only the nodes reachable from `root` through cached child links (every node the searches below the current root
// have walked to) and slide them, with their edges, to the front of the pools; rebuild the hash table.  The reference
// never frees tree entries during a game (player.py:49, self_play.py:107); this is what the engine does INSTEAD of
// dropping the whole table when a pool cannot hold the next search.  Statistics of every kept node are untouched.
// Positions that were only reachable by transposition through an edge never walked from the kept subtree are dropped
// and would be re-expanded if met again.  Returns the new root index.
CZ_D int game_compact(const EngineDev& E, int g, int root) {
  const int nn = E.n_nodes[g];
  int32_t* map = E.gc_map + (size_t)g * E.ncap;
  uint32_t* queue = E.hash + (size_t)g * E.hcap;            // the table is rebuilt below; borrow it as the BFS queue
  czs::syncwarp();
  for (int i = czs::lane(); i < nn; i += 32) map[i] = 0;
  czs::syncwarp();
  if (czs::lane() == 0) {                                    // breadth-first walk over child links
    int head = 0, tail = 0;
    queue[tail++] = (uint32_t)root; map[root] = 1;
    while (head < tail) {
      const int n = (int)queue[head++];
      const size_t ni = (size_t)g * E.ncap + n;
      const int L = (int)(E.node_meta[ni] & 0xff);
      const size_t eo = (size_t)g * E.ecap + E.node_edge_off[ni];
      for (int i = 0; i < L; ++i) {
        const int c = E.edge_child[eo + i];
        if (c >= 0 && map[c] == 0) { map[c] = 1; queue[tail++] = (uint32_t)c; }
      }
    }
  }
  czs::syncwarp();
  // new indices in old order (so every move below goes towards lower addresses)
  int cnt = 0;
  for (int base = 0; base < nn; base += 32) {
    const int i = base + czs::lane();
    const bool k = i < nn && map[i] != 0;
    const unsigned m = czs::ballot(k);
    if (k) map[i] = cnt + czs::popc(m & ((1u << czs::lane()) - 1u)) + 1;
    cnt += czs::popc(m);
  }
  czs::syncwarp();
  // slide nodes and their edges
  int ne = 0;
  for (int i = 0; i < nn; ++i) {
    const int j1 = map[i];
    if (j1 == 0) continue;
    const int j = j1 - 1;
    const size_t si = (size_t)g * E.ncap + i, di = (size_t)g * E.ncap + j;
    const int L = (int)(E.node_meta[si] & 0xff);
    const size_t so = (size_t)g * E.ecap + E.node_edge_off[si], dof = (size_t)g * E.ecap + ne;
    czs::syncwarp();
    for (int b = 0; b < L; b += 32) {
      const int k = b + czs::lane();
      int n_ = 0, ch = 0; double w_ = 0; float p_ = 0; uint16_t mv = 0;
      if (k < L) { n_ = E.edge_n[so + k]; w_ = E.edge_w[so + k]; p_ = E.edge_p[so + k]; mv = E.edge_move[so + k]; ch = E.edge_child[so + k]; }
      czs::syncwarp();
      if (k < L) {
        if (ch >= 0) ch = map[ch] ? map[ch] - 1 : CHILD_UNKNOWN;
        E.edge_n[dof + k] = n_; E.edge_w[dof + k] = w_; E.edge_p[dof + k] = p_; E.edge_move[dof + k] = mv; E.edge_child[dof + k] = ch;
      }
      czs::syncwarp();
    }
    if (czs::lane() == 0) {
      const uint64_t k0 = E.node_key0[si], k1 = E.node_key1[si];
      const int sn = E.node_sum_n[si]; const uint32_t meta = E.node_meta[si]; const float nv = E.node_v[si];
      E.node_key0[di] = k0; E.node_key1[di] = k1; E.node_sum_n[di] = sn; E.node_meta[di] = meta; E.node_edge_off[di] = (uint32_t)ne;
      E.node_v[di] = nv;
    }
    ne += L;
    czs::syncwarp();
  }
  // rebuild the table
  uint32_t* h = E.hash + (size_t)g * E.hcap;
  for (int i = czs::lane(); i < E.hcap; i += 32) h[i] = 0;
  czs::syncwarp();
  if (czs::lane() == 0) {
    const uint32_t mask = (uint32_t)E.hcap - 1;
    for (int j = 0; j < cnt; ++j) {
      uint32_t s = (uint32_t)E.node_key0[(size_t)g * E.ncap + j] & mask;
      while (h[s] != 0) s = (s + 1) & mask;
      h[s] = (uint32_t)j + 1;
    }
    E.n_nodes[g] = cnt; E.n_edges[g] = ne;
#if defined(CZ_EMUL)
    E.counters[5] += 1;
#else
    atomicAdd(E.counters + 5, 1ULL);
#endif
  }
  czs::syncwarp();
  return map[root] - 1;
}

// ------------------------------------------------------------------ begin: tree reuse and task count (action, :147-171)
// raw_tasks: run exactly sims_override simulations (the caller did the bookkeeping of player.py:153-165 itself)
CZ_D void game_begin(const EngineDev& E, int g, int sims_override, bool raw_tasks, TreeSmem* sm) {
  if (!E.active[g]) return;
  copy_board(E.root_board + (size_t)g * BOARD_STRIDE, sm->board);
  uint64_t k0, k1;
  board_key(sm->board, &k0, &k1);
  int root = tt_lookup(E, g, k0, k1);
  const int sims = E.sp.sims_game[g] > 0 ? E.sp.sims_game[g] : E.sims;   // play_config.simulation_num_per_move of this game
  int done = root >= 0 ? E.node_sum_n[(size_t)g * E.ncap + root] : 0;
  if (E.n_no_act[g] > 0 || E.increase_temp[g] || done == sims) done = 0;
  int num_task = sims - done;
  if (sims_override > 0) num_task = sims_override > done ? sims_override - done : 0;
  if (raw_tasks) num_task = sims_override;
  if (num_task < 0) num_task = 0;
  // pools must be able to hold this search; otherwise start from an empty table (counted)
  bool low = (E.ncap - E.n_nodes[g] < num_task + 2 || E.ecap - E.n_edges[g] < (num_task + 2) * 64) && E.n_nodes[g] > 0;
  czs::syncwarp();                                   // reads above complete before lane 0 rewrites the counters
  if (low && root >= 0) {                            // keep what the game can still reach, drop the rest
    root = game_compact(E, g, root);
    low = E.ncap - E.n_nodes[g] < num_task + 2 || E.ecap - E.n_edges[g] < (num_task + 2) * 64;
    czs::syncwarp();
  }
  if (low) {
    uint32_t* h = E.hash + (size_t)g * E.hcap;
    for (int i = czs::lane(); i < E.hcap; i += 32) h[i] = 0;
    if (czs::lane() == 0) {
      E.n_nodes[g] = 0; E.n_edges[g] = 0;
#if defined(CZ_EMUL)
      E.counters[4] += 1;
#else
      atomicAdd(E.counters + 4, 1ULL);
#endif
    }
    czs::syncwarp();
    root = -1;
    num_task = sims_override > 0 ? sims_override : sims;
    if (raw_tasks) num_task = sims_override > 0 ? sims_override : 0;
  }
  if (czs::lane() == 0) {
    E.root_node[g] = root;
    E.tasks_left[g] = num_task;
    E.round_pending[g] = 0;
    E.sims_run[g] = 0;
    E.noise_used[g] = 0;
    E.noise_epoch[g] += 1;
    E.n_leaf[g] = 0; E.n_park[g] = 0; E.n_resume[g] = 0;
  }
  czs::syncwarp();
}

// print_depth_info (player.py:408-450): the most visited line from the root.  At every node the LAST edge with the
// largest N wins (`>=`, :421), the root skips no_act moves; the walk stops at a position that is not in the tree or was
// never selected through (`len(node.a) == 0`, :418), or after max_len plies.  out_moves: canonical moves of the side to
// move at each ply.  *out_value / *out_has_value: `debug[state]` of the position the walk ended on (:436-437).
CZ_D int game_pv(const EngineDev& E, int g, int max_len, uint16_t* out_moves, float* out_value, int* out_has_value, TreeSmem* sm) {
  copy_board(E.root_board + (size_t)g * BOARD_STRIDE, sm->board);
  uint64_t k0, k1;
  board_key(sm->board, &k0, &k1);
  int node = tt_lookup(E, g, k0, k1);
  int len = 0;
  bool root = true;
  while (len < max_len) {
    if (node < 0) break;
    const size_t ni = (size_t)g * E.ncap + node;
    if (E.node_sum_n[ni] < 2) break;                 // expanded but never selected through: node.a is still empty
    const int L = (int)(E.node_meta[ni] & 0xff);
    const size_t eo = (size_t)g * E.ecap + E.node_edge_off[ni];
    int best = -1, n = 0;
    if (czs::lane() == 0) {
      for (int i = 0; i < L; ++i) {
        const int en = E.edge_n[eo + i];
        if (en >= n) {
          bool banned = false;
          if (root) for (int k = 0; k < E.n_no_act[g]; ++k) banned |= E.no_act[(size_t)g * CZ_MAX_NO_ACT + k] == E.edge_move[eo + i];
          if (banned) continue;
          n = en; best = i;
        }
      }
    }
    best = czs::shfl(best, 0);
    if (best < 0) break;
    const move_t mv = E.edge_move[eo + best];
    if (czs::lane() == 0) out_moves[len] = mv;
    ++len;
    step_flip(sm->board, mv, sm->board);
    board_key(sm->board, &k0, &k1);
    node = tt_lookup(E, g, k0, k1);
    root = false;
  }
  if (czs::lane() == 0) {
    const bool has = node >= 0 && !(E.node_meta[(size_t)g * E.ncap + node] & NODE_WAITING);
    *out_has_value = has ? 1 : 0;
    *out_value = has ? E.node_v[(size_t)g * E.ncap + node] : 0.f;
  }
  czs::syncwarp();
  return len;
}

}  // namespace cz
