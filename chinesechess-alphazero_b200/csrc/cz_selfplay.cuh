// cz_selfplay.cuh — the per-ply game loop of worker/self_play.py:95-212 on the device, one warp per game:
// calc_policy + apply_temperature + sampling (agent/player.py:375-406,453-470,195), new_step, the draw /
// repetition / resign adjudication (self_play.py:126-175), the final king capture and value signs
// (:177-191), the store rule (:194-200) and the play record (:202-208).
#pragma once
#include "cz_tree.cuh"

namespace cz {

enum { REC_RESIGN = 1, REC_DRAW_RULE = 2, REC_NOT_STORED = 4 };

template <class CarverT, class CfgT>
inline void selfplay_carve(SelfplayDev& sp, CarverT& cv, const CfgT& c) {
  const size_t G = c.n_games, S = (size_t)c.max_plies + 4;
  sp.hist_stride = (int32_t)S;
  sp.turns = cv.template take<int32_t>(G); sp.no_eat = cv.template take<int32_t>(G);
  sp.enable_resign = cv.template take<int32_t>(G); sp.games_started = cv.template take<int32_t>(G);
  sp.sims_game = cv.template take<int32_t>(G); sp.retired = cv.template take<int32_t>(G);
  sp.game_quota = c.game_quota; sp.playouts_lo = c.playouts_lo; sp.playouts_hi = c.playouts_hi;
  sp.hist_k0 = cv.template take<uint64_t>(G * S); sp.hist_k1 = cv.template take<uint64_t>(G * S);
  sp.hist_move = cv.template take<uint16_t>(G * S);
  sp.rec_cap = (int32_t)(2 * G < 64 ? 64 : 2 * G);
  sp.rec_hdr = cv.template take<RecordHdr>((size_t)sp.rec_cap);
  sp.rec_moves = cv.template take<uint16_t>((size_t)sp.rec_cap * S);
  sp.rec_count = cv.template take<int32_t>(4);
  sp.finished = sp.rec_count + 1;
  sp.enable_resign_rate = c.enable_resign_rate;
}

// cz_config.record_visits, carved after everything else so that no other buffer moves.  Staging holds the worst case of a
// game (every ply with MAX_MOVES visited edges), the heap that of a full ring, so the heap cannot overflow while the ring
// has a slot.  The heap side is one block: [pairs used u64][first pair per record i64 x rec_cap][pairs per ply u8 x
// rec_cap x hist_stride, padded to 8][pairs (label, N) u32 x 2].
inline size_t visits_pairs_cap(const SelfplayDev& sp) { return (size_t)sp.rec_cap * sp.hist_stride * MAX_MOVES; }
inline size_t visits_cnt_off(const SelfplayDev& sp) { return 8 + 8 * (size_t)sp.rec_cap; }
inline size_t visits_heap_off(const SelfplayDev& sp) { return (visits_cnt_off(sp) + (size_t)sp.rec_cap * sp.hist_stride + 7) & ~(size_t)7; }
inline size_t visits_block_bytes(const SelfplayDev& sp) { return visits_heap_off(sp) + 8 * visits_pairs_cap(sp); }

template <class CarverT, class CfgT>
inline void visits_carve(SelfplayDev& sp, CarverT& cv, const CfgT& c) {
  sp.record_visits = c.record_visits ? 1 : 0;
  if (!sp.record_visits) return;
  const size_t G = c.n_games, S = sp.hist_stride;
  sp.vis_lab = cv.template take<uint16_t>(G * S * MAX_MOVES); sp.vis_n = cv.template take<uint32_t>(G * S * MAX_MOVES);
  sp.vis_ply = cv.template take<uint8_t>(G * S); sp.vis_cursor = cv.template take<int32_t>(G);
  uint8_t* blk = cv.template take<uint8_t>(visits_block_bytes(sp));
  sp.vis_used = reinterpret_cast<unsigned long long*>(blk);
  sp.rec_vis_off = reinterpret_cast<int64_t*>(blk ? blk + 8 : nullptr);
  sp.rec_vis_cnt = blk ? blk + visits_cnt_off(sp) : nullptr;
  sp.vis_heap = reinterpret_cast<uint32_t*>(blk ? blk + visits_heap_off(sp) : nullptr);
}

// The root's (label, N) pairs of ply `ply` appended to the game's staging, in ascending label order: every edge with
// N > 0, which excludes the no_act moves (calc_policy zeroes them, player.py:381-383).  Only reads the search's state.
CZ_D void record_root_visits(const SelfplayDev& sp, int g, int ply, const int nv[4], const int lab[4], int L) {
  int key[4], rank[4];
  for (int c = 0; c < 4; ++c) { key[c] = nv[c] > 0 && lab[c] >= 0 ? lab[c] : 0x7fffffff; rank[c] = 0; }
  for (int j = 0; j < L; ++j) {                     // all lanes walk the same j: broadcast via shfl
    const int oc = j >> 5;
    const int ok = czs::shfl(oc == 0 ? key[0] : oc == 1 ? key[1] : oc == 2 ? key[2] : key[3], j & 31);
    for (int c = 0; c < 4; ++c) rank[c] += ok < key[c] ? 1 : 0;
  }
  int kept = 0;
  for (int c = 0; c < 4; ++c) kept += key[c] != 0x7fffffff ? 1 : 0;
  kept = czs::warp_sum(kept);
  const size_t base = (size_t)g * sp.hist_stride * MAX_MOVES + sp.vis_cursor[g];
  for (int c = 0; c < 4; ++c)
    if (key[c] != 0x7fffffff) { sp.vis_lab[base + rank[c]] = (uint16_t)key[c]; sp.vis_n[base + rank[c]] = (uint32_t)nv[c]; }
  czs::syncwarp();
  if (czs::lane() == 0) { sp.vis_ply[(size_t)g * sp.hist_stride + ply] = (uint8_t)kept; sp.vis_cursor[g] += kept; }
  czs::syncwarp();
}

// (Re)start the game in slot g at the position currently in root_board: fresh history, counters and
// the per-game resign lottery (`random() > enable_resign_rate`, self_play.py:102-105).
CZ_D void selfplay_start_game(const EngineDev& E, int g, uint8_t* board_smem) {
  const SelfplayDev& sp = E.sp;
  copy_board(E.root_board + (size_t)g * BOARD_STRIDE, board_smem);
  uint64_t k0, k1;
  board_key(board_smem, &k0, &k1);
  if (czs::lane() == 0) {
    const int idx = sp.games_started[g];
    Rng r; r.init(E.seed, E.rank, (uint32_t)g, 3u, (uint32_t)idx);
    sp.enable_resign[g] = r.uniform() > sp.enable_resign_rate ? 1 : 0;
    sp.turns[g] = 0; sp.no_eat[g] = 0;
    if (sp.record_visits) sp.vis_cursor[g] = 0;
    // evaluator.py:153-154: `playouts = randint(8, 12) * 100` once per game; both player slots of a game draw the same value
    int sg = 0;
    if (E.arena && sp.playouts_lo > 0 && sp.playouts_hi >= sp.playouts_lo) {
      Rng q; q.init(E.seed, E.rank, (uint32_t)(g % (E.n_games / 2)), 5u, (uint32_t)idx);
      sg = (sp.playouts_lo + (int)(q.next() % (uint32_t)(sp.playouts_hi - sp.playouts_lo + 1))) * 100;
    }
    sp.sims_game[g] = sg;
    sp.hist_k0[(size_t)g * sp.hist_stride] = k0;
    sp.hist_k1[(size_t)g * sp.hist_stride] = k1;
  }
  czs::syncwarp();
}

// Arena (worker/evaluator.py:147-170): slots g and partner(g) are the two players' trees of game (g mod M).  The game with
// running index idx = started*M + (g mod M) has player idx % 2 as red ("even: best = red, odd: best = black"); only the
// slot of the player to move is active.
CZ_D int arena_partner(const EngineDev& E, int g) { const int m = E.n_games / 2; return g < m ? g + m : g - m; }
CZ_D int arena_mover_slot(const EngineDev& E, int g, int started, int turns) {
  const int m = E.n_games / 2, i = g % m;
  const int idx = started * m + i;
  const int player = (idx + turns) & 1;             // red = player idx % 2 moves on even plies
  return i + player * m;
}

// running index of the game a slot plays after `started` earlier ones: the i-th of M (arena) / G concurrent games
CZ_D int game_index_of(const EngineDev& E, int g, int started) {
  return E.arena ? started * (E.n_games / 2) + g % (E.n_games / 2) : started * E.n_games + g;
}

CZ_D void selfplay_reset_game(const EngineDev& E, int g) {
  if (czs::lane() == 0) { E.sp.games_started[g] = 0; E.sp.retired[g] = 0; }
  czs::syncwarp();
  TreeSmem* sm = reinterpret_cast<TreeSmem*>(czs::dyn_smem()) + czs::warp_in_block();
  selfplay_start_game(E, g, sm->board);
  if (E.arena && czs::lane() == 0) {
    E.sp.enable_resign[g] = 0;                      // evaluator.py:157-160: enable_resign=False
    E.active[g] = arena_mover_slot(E, g, 0, 0) == g ? 1 : 0;
  }
  if (E.sp.game_quota > 0 && game_index_of(E, g, 0) >= E.sp.game_quota && czs::lane() == 0) {   // more slots than games
    E.sp.retired[g] = 1; E.active[g] = 0;
  }
  czs::syncwarp();
}

// After slot g played a ply (game not over): hand the game to the partner slot — same position, counters, history and the
// bans computed for the next mover — and flip which of the two is active.
CZ_D void arena_handover(const EngineDev& E, int g, int turns_before, int turns_after) {
  const SelfplayDev& sp = E.sp;
  const int p = arena_partner(E, g);
  czs::syncwarp();
  for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) E.root_board[(size_t)p * BOARD_STRIDE + k] = E.root_board[(size_t)g * BOARD_STRIDE + k];
  if (czs::lane() == 0) {
    sp.turns[p] = sp.turns[g]; sp.no_eat[p] = sp.no_eat[g];
    const size_t hg = (size_t)g * sp.hist_stride, hp = (size_t)p * sp.hist_stride;
    for (int t = turns_before; t < turns_after; ++t) sp.hist_move[hp + t] = sp.hist_move[hg + t];
    for (int t = turns_before + 1; t <= turns_after; ++t) { sp.hist_k0[hp + t] = sp.hist_k0[hg + t]; sp.hist_k1[hp + t] = sp.hist_k1[hg + t]; }
    const int n = E.n_no_act[g];
    E.n_no_act[p] = n;
    for (int k = 0; k < n; ++k) E.no_act[(size_t)p * CZ_MAX_NO_ACT + k] = E.no_act[(size_t)g * CZ_MAX_NO_ACT + k];
    E.increase_temp[p] = E.increase_temp[g];
    E.n_no_act[g] = 0; E.increase_temp[g] = 0;
    E.active[g] = 0; E.active[p] = 1;
  }
  czs::syncwarp();
}

CZ_D void clear_tree(const EngineDev& E, int g) {
  uint32_t* h = E.hash + (size_t)g * E.hcap;
  for (int i = czs::lane(); i < E.hcap; i += 32) h[i] = 0;
  if (czs::lane() == 0) { E.n_nodes[g] = 0; E.n_edges[g] = 0; E.root_node[g] = -1; }
  czs::syncwarp();
}

// One ply of game g after its search finished.
CZ_D void game_play(const EngineDev& E, int g, const uint8_t* init_board, TreeSmem* sm) {
  const SelfplayDev& sp = E.sp;
  if (!E.active[g]) return;
  const int root = E.root_node[g];
  if (root < 0) return;
  const size_t ni = (size_t)g * E.ncap + root;
  const int L = (int)(E.node_meta[ni] & 0xff);
  const size_t eo = (size_t)g * E.ecap + E.node_edge_off[ni];
  const int turns0 = sp.turns[g];
  const int nna = E.n_no_act[g];
  const uint16_t* na = E.no_act + (size_t)g * CZ_MAX_NO_ACT;
  // ---- calc_policy (player.py:375-406): visit counts, resign test on the best q
  double sum_n = 0.0, max_q = -100.0;
  int nv[4], lab[4]; bool ban[4];
  for (int c = 0; c < 4; ++c) {
    const int i = c * 32 + czs::lane();
    nv[c] = 0; lab[c] = 0x7fffffff; ban[c] = true;
    if (i < L) {
      const move_t m = E.edge_move[eo + i];
      bool b = false;
      for (int k = 0; k < nna; ++k) b = b || na[k] == m;
      ban[c] = b;
      lab[c] = E.label_lut[mv_from(m) * 90 + mv_to(m)];
      if (!b) {
        nv[c] = E.edge_n[eo + i];
        const double q = nv[c] != 0 ? E.edge_w[eo + i] / (double)nv[c] : 0.0;
        if (q > max_q) max_q = q;
      }
    }
  }
  for (int m = 16; m; m >>= 1) { const double o = czs::shfl_xor(max_q, m); max_q = o > max_q ? o : max_q; }
  { int s = nv[0] + nv[1] + nv[2] + nv[3]; s = czs::warp_sum(s); sum_n = (double)s; }
  const bool resign = max_q < E.resign_threshold && sp.enable_resign[g] && turns0 > E.min_resign_turn;

  int value = 0, flags = 0;
  bool over = false;
  int turns = turns0;
  int final_from_to = -1;
  if (resign) {
    value = -1; over = true; flags |= REC_RESIGN;
  } else {
    // ---- apply_temperature (player.py:453-470) and np.random.choice (:195), labels in index order
    double tau = 0.0;
    if (turns0 < 30 && E.tau_decay != 0.0) tau = pow(E.tau_decay, (double)(turns0 + 1));
    if (tau < 0.1) tau = 0.0;
    if (E.increase_temp[g]) tau = 0.5;
    double wgt[4];
    for (int c = 0; c < 4; ++c) {
      wgt[c] = 0.0;
      if (nv[c] > 0) wgt[c] = tau == 0.0 ? (double)nv[c] : pow((double)nv[c] / sum_n, 1.0 / tau);
    }
    int chosen = -1;
    if (tau == 0.0) {                               // argmax, first maximum in label order
      double bw = -1.0; int bl = 0x7fffffff, bi = -1;
      for (int c = 0; c < 4; ++c)
        if (!ban[c] && lab[c] != 0x7fffffff && (wgt[c] > bw || (wgt[c] == bw && lab[c] < bl))) { bw = wgt[c]; bl = lab[c]; bi = c * 32 + czs::lane(); }
      for (int m = 16; m; m >>= 1) {
        const double ow = czs::shfl_xor(bw, m); const int ol = czs::shfl_xor(bl, m), oi = czs::shfl_xor(bi, m);
        if (oi >= 0 && (bi < 0 || ow > bw || (ow == bw && ol < bl))) { bw = ow; bl = ol; bi = oi; }
      }
      chosen = bi;
    } else {
      double tot = wgt[0] + wgt[1] + wgt[2] + wgt[3];
      for (int m = 16; m; m >>= 1) tot += czs::shfl_xor(tot, m);
      Rng r; r.init(E.seed, E.rank, (uint32_t)g, 2u, (uint32_t)(sp.games_started[g] * 1024 + turns0));
      const double u = r.uniform() * tot;
      // cumulative weight of all edges with a smaller label than mine
      double best_c = 1e300; int bi = -1, fallback = -1; double fb_l = -1.0;
      for (int c = 0; c < 4; ++c) {
        const int i = c * 32 + czs::lane();
        double before = 0.0;
        for (int j = 0; j < L; ++j) {                 // all lanes walk the same j: broadcast via shfl
          const int oc = j >> 5, ol = j & 31;
          const double ow = czs::shfl(oc == 0 ? wgt[0] : oc == 1 ? wgt[1] : oc == 2 ? wgt[2] : wgt[3], ol);
          const int olab = czs::shfl(oc == 0 ? lab[0] : oc == 1 ? lab[1] : oc == 2 ? lab[2] : lab[3], ol);
          if (olab < lab[c]) before += ow;
        }
        if (i < L && wgt[c] > 0.0) {
          if (before + wgt[c] > u && before < best_c) { best_c = before; bi = i; }   // first label whose cdf exceeds u
          if ((double)lab[c] > fb_l) { fb_l = (double)lab[c]; fallback = i; }
        }
      }
      for (int m = 16; m; m >>= 1) {
        const double oc = czs::shfl_xor(best_c, m); const int oi = czs::shfl_xor(bi, m);
        if (oi >= 0 && (bi < 0 || oc < best_c)) { best_c = oc; bi = oi; }
        const double ofl = czs::shfl_xor(fb_l, m); const int ofi = czs::shfl_xor(fallback, m);
        if (ofi >= 0 && (fallback < 0 || ofl > fb_l)) { fb_l = ofl; fallback = ofi; }
      }
      chosen = bi >= 0 ? bi : fallback;
    }
    if (chosen < 0) {                               // no visits at all: cannot happen after a search
      if (czs::lane() == 0) E.game_err[g] |= GAME_ERR_NOMOVE;
      chosen = 0;
    }
    const move_t mv = E.edge_move[eo + chosen];
    if (sp.record_visits) record_root_visits(sp, g, turns0, nv, lab, L);
    // ---- play it (self_play.py:132-147)
    copy_board(E.root_board + (size_t)g * BOARD_STRIDE, sm->board);
    const bool no_eat = step_flip(sm->board, mv, sm->board);
    if (czs::lane() == 0) sp.hist_move[(size_t)g * sp.hist_stride + turns] = mv;
    ++turns;
    const int nec = no_eat ? sp.no_eat[g] + 1 : 0;
    uint64_t k0, k1;
    board_key(sm->board, &k0, &k1);
    if (czs::lane() == 0) {
      sp.no_eat[g] = nec;
      sp.hist_k0[(size_t)g * sp.hist_stride + turns] = k0;
      sp.hist_k1[(size_t)g * sp.hist_stride + turns] = k1;
      E.n_no_act[g] = 0; E.increase_temp[g] = 0;
    }
    czs::syncwarp();
    if (nec >= 120 || turns >= 2 * E.max_game_length) {          // :149-151
      over = true; value = 0; flags |= REC_DRAW_RULE;
    } else {
      int nm;
      const DoneResult dr = done_eval(sm->board, sm->list, &nm, true, sm->sc.b0, sm->sc.l0);
      over = dr.over != 0; value = dr.v;
      if (dr.final_move >= 0) final_from_to = sm->list[dr.final_move];
      if (!over && !has_attack_chessman(sm->board)) { over = true; value = 0; flags |= REC_DRAW_RULE; }   // :155-158
      if (!over && !dr.check) {
        // repetition handling (:161-175): earlier occurrences of this state, oldest first
        int n_ban = 0, idle = 0; bool inc = false;
        for (int i = 0; i < turns && !over; ++i) {
          const size_t hi = (size_t)g * sp.hist_stride + i;
          if (sp.hist_k0[hi] != k0 || sp.hist_k1[hi] != k1) continue;
          const move_t pm = sp.hist_move[hi];
          if (E.arena) inc = true;                   // evaluator.py:176-178: any repetition raises the temperature
          if (will_check_or_catch(sm->board, pm, &sm->sc)) {
            if (n_ban < CZ_MAX_NO_ACT) { if (czs::lane() == 0) E.no_act[(size_t)g * CZ_MAX_NO_ACT + n_ban] = pm; ++n_ban; }
          } else if (E.arena || !be_catched(sm->board, pm, &sm->sc)) {   // the evaluator has no be_catched exemption (:186-193)
            inc = true;
            if (++idle >= 3) { over = true; value = 0; flags |= REC_DRAW_RULE; }
          }
        }
        if (czs::lane() == 0) { E.n_no_act[g] = n_ban; E.increase_temp[g] = inc ? 1 : 0; }
        czs::syncwarp();
      }
    }
    if (over && final_from_to >= 0) {                // the king capture is appended to the record (:177-184)
      if (czs::lane() == 0) {
        sp.hist_move[(size_t)g * sp.hist_stride + turns] = (uint16_t)final_from_to;
        if (sp.record_visits) sp.vis_ply[(size_t)g * sp.hist_stride + turns] = 0;     // never searched
      }
      ++turns;
      value = -value;
    }
  }
  if (!over) {
    // next root = the new state; the tree is kept (same player object, self_play.py:107,124)
    for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) E.root_board[(size_t)g * BOARD_STRIDE + k] = k < NSQ ? sm->board[k] : (uint8_t)0;
    if (czs::lane() == 0) sp.turns[g] = turns;
    czs::syncwarp();
    if (E.arena) arena_handover(E, g, turns0, turns);
    return;
  }
  // ---- game over: result from red's view (:190-191), store rule (:194-200), record (:202-208)
  if (turns % 2 == 1) value = -value;
  bool store = true;
  if (turns < 10 && !E.arena) {
    Rng r; r.init(E.seed, E.rank, (uint32_t)g, 4u, (uint32_t)sp.games_started[g]);
    store = r.uniform() > 0.9;
  }
  int slot = -1;
  if (czs::lane() == 0) {
#if defined(CZ_EMUL)
    slot = sp.rec_count[0]; sp.rec_count[0] = slot + 1; sp.finished[0] += 1;
#else
    slot = atomicAdd(sp.rec_count, 1); atomicAdd(sp.finished, 1);
#endif
  }
  slot = czs::shfl(slot, 0);
  if (slot >= sp.rec_cap && czs::lane() == 0) {      // ring full: counted, never silent (cz_get_counters [3])
#if defined(CZ_EMUL)
    E.counters[3] += 1;
#else
    atomicAdd(E.counters + 3, 1ULL);
#endif
  }
  if (slot < sp.rec_cap) {
    if (czs::lane() == 0) {
      RecordHdr h; h.n_plies = turns; h.value_red = value;
      h.game_index = game_index_of(E, g, sp.games_started[g]);
      h.flags = flags | (store ? 0 : REC_NOT_STORED);
      sp.rec_hdr[slot] = h;
    }
    for (int i = czs::lane(); i < turns; i += 32)
      sp.rec_moves[(size_t)slot * sp.hist_stride + i] = sp.hist_move[(size_t)g * sp.hist_stride + i];
    if (sp.record_visits) {                          // the staged pairs into the heap, claimed like the ring slot
      const int np = sp.vis_cursor[g];
      unsigned long long off = 0;
      if (czs::lane() == 0) {
#if defined(CZ_EMUL)
        off = sp.vis_used[0]; sp.vis_used[0] = off + (unsigned long long)np;
#else
        off = atomicAdd(sp.vis_used, (unsigned long long)np);
#endif
        sp.rec_vis_off[slot] = (int64_t)off;
      }
      off = czs::shfl(off, 0);
      const size_t src = (size_t)g * sp.hist_stride;
      for (int i = czs::lane(); i < turns; i += 32) sp.rec_vis_cnt[(size_t)slot * sp.hist_stride + i] = sp.vis_ply[src + i];
      for (int i = czs::lane(); i < np; i += 32) {
        sp.vis_heap[2 * (off + i)] = sp.vis_lab[src * MAX_MOVES + i];
        sp.vis_heap[2 * (off + i) + 1] = sp.vis_n[src * MAX_MOVES + i];
      }
    }
  }
  // ---- quota reached: the slot (both player slots of an arena game) retires with an empty tree
  if (sp.game_quota > 0 && game_index_of(E, g, sp.games_started[g] + 1) >= sp.game_quota) {
    if (czs::lane() == 0) { sp.retired[g] = 1; E.active[g] = 0; E.n_no_act[g] = 0; E.increase_temp[g] = 0; }
    czs::syncwarp();
    clear_tree(E, g);
    if (E.arena) {
      const int p = arena_partner(E, g);
      if (czs::lane() == 0) { sp.retired[p] = 1; E.active[p] = 0; E.n_no_act[p] = 0; E.increase_temp[p] = 0; }
      czs::syncwarp();
      clear_tree(E, p);
    }
    return;
  }
  // ---- restart the slot from the initial position with an empty tree
  for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) E.root_board[(size_t)g * BOARD_STRIDE + k] = k < NSQ ? init_board[k] : (uint8_t)0;
  if (czs::lane() == 0) { sp.games_started[g] += 1; E.n_no_act[g] = 0; E.increase_temp[g] = 0; }
  czs::syncwarp();
  clear_tree(E, g);
  selfplay_start_game(E, g, sm->board);
  if (E.arena) {                                     // both players start the next game of this pair with empty trees
    const int p = arena_partner(E, g);
    for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) E.root_board[(size_t)p * BOARD_STRIDE + k] = k < NSQ ? init_board[k] : (uint8_t)0;
    if (czs::lane() == 0) { sp.games_started[p] = sp.games_started[g]; E.n_no_act[p] = 0; E.increase_temp[p] = 0; }
    czs::syncwarp();
    clear_tree(E, p);
    selfplay_start_game(E, p, sm->board);
    if (czs::lane() == 0) {
      sp.enable_resign[g] = 0; sp.enable_resign[p] = 0;
      const int mv = arena_mover_slot(E, g, sp.games_started[g], 0);
      E.active[g] = mv == g ? 1 : 0; E.active[p] = mv == p ? 1 : 0;
    }
    czs::syncwarp();
  }
}

}  // namespace cz
