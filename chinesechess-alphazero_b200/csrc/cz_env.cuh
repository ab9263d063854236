// cz_env.cuh — Xiangqi rules on packed boards, warp-cooperative device functions.
//
// Replaces (bit-exact) the string-based rules engine of the reference:
//   cchess_alphazero/environment/static_env.py  (get_legal_moves :256-321, done :14-77,
//   step/new_step :79-98, fliped_state :245-254, state_to_planes :137-156,
//   will_check_or_catch :390-421, get_catch_list :423-454, be_catched :456-469,
//   has_attack_chessman :471-479) and light_env/common.py mov_dir :66-76.
//
// Board: 90 bytes, sq = y*9 + x, y = 0 is the side-to-move's back rank (the reference's
// internal board[y][x]); every position is stored from the side to move ("canonical").
// Piece code: 0 empty, 1..7 side-to-move P C R N E A K, 9..15 opponent (bit 3 = opponent).
// The type order is the plane order of lookup_tables.py Fen_2_Idx :27-42, so
// plane = code-1 (own) / code-2 (opponent), plane row = 9 - y.
// Move: uint16 (from << 8) | to.  One warp owns one board; all functions below must be
// called by all 32 lanes with warp-uniform arguments.
#pragma once
#include "cz_simt.h"

namespace cz {

typedef uint16_t move_t;
enum { NSQ = 90, BOARD_STRIDE = 96, MAX_MOVES = 128, N_LABELS = 2086 };
enum : uint8_t { PC_EMPTY = 0, PC_P = 1, PC_C = 2, PC_R = 3, PC_N = 4, PC_E = 5, PC_A = 6, PC_K = 7, PC_OPP = 8 };

CZ_HD bool pc_own(uint8_t c) { return c != 0 && (c & 8) == 0; }
CZ_HD bool pc_opp(uint8_t c) { return (c & 8) != 0; }
CZ_HD int mv_from(move_t m) { return m >> 8; }
CZ_HD int mv_to(move_t m) { return m & 0xff; }
CZ_HD move_t mv_make(int f, int t) { return (move_t)((f << 8) | t); }

// ------------------------------------------------------------------ per-piece generation
// can_move (static_env.py:323-330): on board and not occupied by the mover's own piece.
CZ_D bool can_move(const uint8_t* b, int x, int y) {
  if (x < 0 || x > 8 || y < 0 || y > 9) return false;
  return !pc_own(b[y * 9 + x]);
}

// Emits the pseudo-legal destinations of the own piece `c` on `sq` in the reference order.
template <class Sink>
CZ_D void gen_piece(const uint8_t* b, int sq, uint8_t c, Sink& out) {
  const int x = sq % 9, y = sq / 9;
  if (c == PC_R || c == PC_C) {
    // x_board_from / y_board_from (static_env.py:332-348): nearest occupied square each way
    int l = x - 1, r = x + 1, d = y - 1, u = y + 1;
    while (l > -1 && b[y * 9 + l] == 0) --l;
    while (r < 9 && b[y * 9 + r] == 0) ++r;
    while (d > -1 && b[d * 9 + x] == 0) --d;
    while (u < 10 && b[u * 9 + x] == 0) ++u;
    for (int x_ = l + 1; x_ < x; ++x_) out(y * 9 + x_);
    for (int x_ = x + 1; x_ < r; ++x_) out(y * 9 + x_);
    for (int y_ = d + 1; y_ < y; ++y_) out(y_ * 9 + x);
    for (int y_ = y + 1; y_ < u; ++y_) out(y_ * 9 + x);
    if (c == PC_R) {
      if (can_move(b, l, y)) out(y * 9 + l);
      if (can_move(b, r, y)) out(y * 9 + r);
      if (can_move(b, x, d)) out(d * 9 + x);
      if (can_move(b, x, u)) out(u * 9 + x);
    } else {
      // cannon: jump exactly one screen (static_env.py:308-320)
      int l_ = l - 1, r_ = r + 1, d_ = d - 1, u_ = u + 1;
      if (l > -1) { while (l_ > -1 && b[y * 9 + l_] == 0) --l_; }
      if (r < 9) { while (r_ < 9 && b[y * 9 + r_] == 0) ++r_; }
      if (d > -1) { while (d_ > -1 && b[d_ * 9 + x] == 0) --d_; }
      if (u < 10) { while (u_ < 10 && b[u_ * 9 + x] == 0) ++u_; }
      if (can_move(b, l_, y)) out(y * 9 + l_);
      if (can_move(b, r_, y)) out(y * 9 + r_);
      if (can_move(b, x, d_)) out(d_ * 9 + x);
      if (can_move(b, x, u_)) out(u_ * 9 + x);
    }
    return;
  }
  // step pieces, mov_dir order (light_env/common.py:66-76), packed as (dx+2) | (dy+2)<<3
  //   king    (0,-1) (1,0) (0,1) (-1,0)
  //   advisor (-1,-1) (1,-1) (-1,1) (1,1)
  //   eleph.  (-2,-2) (2,-2) (2,2) (-2,2)
  //   knight  (-1,-2) (1,-2) (2,-1) (2,1) (1,2) (-1,2) (-2,1) (-2,-1)
  //   pawn    (0,1) (-1,0) (1,0)
  int nd;
  uint64_t dirs;
#define CZ_DIR(dx, dy) ((uint64_t)(((dx) + 2) | (((dy) + 2) << 3)))
  switch (c) {
    case PC_K: nd = 4; dirs = CZ_DIR(0, -1) | CZ_DIR(1, 0) << 6 | CZ_DIR(0, 1) << 12 | CZ_DIR(-1, 0) << 18; break;
    case PC_A: nd = 4; dirs = CZ_DIR(-1, -1) | CZ_DIR(1, -1) << 6 | CZ_DIR(-1, 1) << 12 | CZ_DIR(1, 1) << 18; break;
    case PC_E: nd = 4; dirs = CZ_DIR(-2, -2) | CZ_DIR(2, -2) << 6 | CZ_DIR(2, 2) << 12 | CZ_DIR(-2, 2) << 18; break;
    case PC_N: nd = 8; dirs = CZ_DIR(-1, -2) | CZ_DIR(1, -2) << 6 | CZ_DIR(2, -1) << 12 | CZ_DIR(2, 1) << 18 |
                             CZ_DIR(1, 2) << 24 | CZ_DIR(-1, 2) << 30 | CZ_DIR(-2, 1) << 36 | CZ_DIR(-2, -1) << 42; break;
    case PC_P: nd = 3; dirs = CZ_DIR(0, 1) | CZ_DIR(-1, 0) << 6 | CZ_DIR(1, 0) << 12; break;
    default: return;
  }
#undef CZ_DIR
  int fly = -1;  // king-faces-king capture square (static_env.py:283-286), same for every step
  if (c == PC_K) {
    int u = y + 1;
    while (u < 10 && b[u * 9 + x] == 0) ++u;
    if (u < 10 && b[u * 9 + x] == (PC_K | PC_OPP)) fly = u * 9 + x;
  }
  for (int i = 0; i < nd; ++i) {
    const int dd = (int)((dirs >> (6 * i)) & 63);
    const int dx = (dd & 7) - 2, dy = (dd >> 3) - 2;
    const int x_ = x + dx, y_ = y + dy;
    if (!can_move(b, x_, y_)) continue;
    if (c == PC_P) {
      if (y < 5 && x_ != x) continue;                // no sideways step before the river
    } else if (c == PC_N || c == PC_E) {
      if (b[(y + dy / 2) * 9 + (x + dx / 2)] != 0) continue;   // leg / eye blocked (C '/' truncates like int())
      if (c == PC_E && y_ > 4) continue;             // elephants stay home
    } else {                                         // king, advisor: palace
      if (x_ < 3 || x_ > 5) continue;
      if (y_ > 2) continue;
    }
    out(y_ * 9 + x_);
    if (fly >= 0) out(fly);
  }
}

struct CountSink { int n; CZ_DM void operator()(int) { ++n; } };
struct EmitSink {
  move_t* list; int pos; int from;
  CZ_DM void operator()(int to) { if (pos < MAX_MOVES) list[pos] = mv_make(from, to); ++pos; }
};

// ------------------------------------------------------------------ occupancy bitboards (movegen)
// The board as bit sets built with six ballots: occ / own over sq = y*9 + x (ranks are 9 consecutive bits) and the same two
// sets transposed, over sqT = x*10 + y (files are 10 consecutive bits).  A sliding piece then finds its blockers with two
// mask operations per direction instead of a dependent shared-memory load per square, and every piece describes its moves
// ONCE (PieceMoves); counting and emitting read the description (gen_piece above walked the board twice per piece).
struct BoardBits { unsigned occ[3], own[3], occT[3], ownT[3]; };
CZ_D unsigned bits96(const unsigned* w, int pos, int n) {       // n <= 16 bits starting at bit `pos` of a 96-bit set
  const int i = pos >> 5, sh = pos & 31;
  const unsigned lo = i == 0 ? w[0] : (i == 1 ? w[1] : w[2]);
  const unsigned hi = i == 0 ? w[1] : (i == 1 ? w[2] : 0u);
  const uint64_t v = (uint64_t)lo | ((uint64_t)hi << 32);
  return (unsigned)(v >> sh) & ((1u << n) - 1u);
}
CZ_D bool bit96(const unsigned* w, int pos) { return bits96(w, pos, 1) != 0u; }
CZ_D void board_bits(const uint8_t* b, BoardBits* bb) {
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    const uint8_t c = sq < NSQ ? b[sq] : (uint8_t)0;
    bb->occ[j] = czs::ballot(c != 0);
    bb->own[j] = czs::ballot(pc_own(c));
    const uint8_t t = sq < NSQ ? b[(sq % 10) * 9 + sq / 10] : (uint8_t)0;      // sqT = x*10 + y  ->  square y*9 + x
    bb->occT[j] = czs::ballot(t != 0);
    bb->ownT[j] = czs::ballot(pc_own(t));
  }
}

// The pseudo-legal moves of one own piece, described once: sliders by their blocker coordinates and capture squares, step
// pieces by a validity mask over their direction table (+ the king's flying-general square).
struct PieceMoves {
  int kind;                 // 0 none, 1 slider (rook / cannon), 2 step piece
  int x, y;
  int l, r, d, u;           // slider: nearest occupied column left / right (-1 / 9), row below / above (-1 / 10)
  int cap[4];               // slider: capture square to the left, right, below, above, or -1
  uint64_t dirs; int nd;    // step piece: direction table (gen_piece's packing) ...
  unsigned valid;           // ... and which entries are playable
  int fly;                  // king: flying-general capture square or -1
  int count;
};
CZ_D int lowest_above(unsigned mask, int i, int none) { const unsigned m = mask >> (i + 1); return m ? i + czs::ffs(m) : none; }
CZ_D int highest_below(unsigned mask, int i) { return czs::fls(mask & ((1u << i) - 1u)) - 1; }      // -1 if none

CZ_D void piece_moves(const uint8_t* b, const BoardBits& bb, int sq, uint8_t c, PieceMoves* pm) {
  pm->kind = 0; pm->count = 0; pm->fly = -1;
  if (sq < 0) return;
  const int x = sq % 9, y = sq / 9;
  pm->x = x; pm->y = y;
  if (c == PC_R || c == PC_C) {
    const unsigned R = bits96(bb.occ, y * 9, 9), F = bits96(bb.occT, x * 10, 10);
    const unsigned Ro = bits96(bb.own, y * 9, 9), Fo = bits96(bb.ownT, x * 10, 10);
    const int l = highest_below(R, x), r = lowest_above(R, x, 9), d = highest_below(F, y), u = lowest_above(F, y, 10);
    pm->kind = 1; pm->l = l; pm->r = r; pm->d = d; pm->u = u;
    int tl = l, tr = r, td = d, tu = u;                                       // rook: the blocker itself
    if (c == PC_C) {                                                          // cannon: the next piece behind the screen
      tl = l > -1 ? highest_below(R, l) : -1;
      tr = r < 9 ? lowest_above(R, r, 9) : 9;
      td = d > -1 ? highest_below(F, d) : -1;
      tu = u < 10 ? lowest_above(F, u, 10) : 10;
    }
    pm->cap[0] = (tl > -1 && !((Ro >> tl) & 1u)) ? y * 9 + tl : -1;
    pm->cap[1] = (tr < 9 && !((Ro >> tr) & 1u)) ? y * 9 + tr : -1;
    pm->cap[2] = (td > -1 && !((Fo >> td) & 1u)) ? td * 9 + x : -1;
    pm->cap[3] = (tu < 10 && !((Fo >> tu) & 1u)) ? tu * 9 + x : -1;
    pm->count = (x - l - 1) + (r - x - 1) + (y - d - 1) + (u - y - 1) + (pm->cap[0] >= 0) + (pm->cap[1] >= 0) + (pm->cap[2] >= 0) + (pm->cap[3] >= 0);
    return;
  }
  int nd;
  uint64_t dirs;
#define CZ_DIR(dx, dy) ((uint64_t)(((dx) + 2) | (((dy) + 2) << 3)))
  switch (c) {
    case PC_K: nd = 4; dirs = CZ_DIR(0, -1) | CZ_DIR(1, 0) << 6 | CZ_DIR(0, 1) << 12 | CZ_DIR(-1, 0) << 18; break;
    case PC_A: nd = 4; dirs = CZ_DIR(-1, -1) | CZ_DIR(1, -1) << 6 | CZ_DIR(-1, 1) << 12 | CZ_DIR(1, 1) << 18; break;
    case PC_E: nd = 4; dirs = CZ_DIR(-2, -2) | CZ_DIR(2, -2) << 6 | CZ_DIR(2, 2) << 12 | CZ_DIR(-2, 2) << 18; break;
    case PC_N: nd = 8; dirs = CZ_DIR(-1, -2) | CZ_DIR(1, -2) << 6 | CZ_DIR(2, -1) << 12 | CZ_DIR(2, 1) << 18 |
                             CZ_DIR(1, 2) << 24 | CZ_DIR(-1, 2) << 30 | CZ_DIR(-2, 1) << 36 | CZ_DIR(-2, -1) << 42; break;
    case PC_P: nd = 3; dirs = CZ_DIR(0, 1) | CZ_DIR(-1, 0) << 6 | CZ_DIR(1, 0) << 12; break;
    default: return;
  }
#undef CZ_DIR
  pm->kind = 2; pm->dirs = dirs; pm->nd = nd;
  if (c == PC_K) {                                            // static_env.py:283-286: the first piece up the file is their king
    const unsigned F = bits96(bb.occT, x * 10, 10);
    const int u = lowest_above(F, y, 10);
    if (u < 10 && b[u * 9 + x] == (PC_K | PC_OPP)) pm->fly = u * 9 + x;
  }
  unsigned valid = 0;
  for (int i = 0; i < nd; ++i) {
    const int dd = (int)((dirs >> (6 * i)) & 63);
    const int dx = (dd & 7) - 2, dy = (dd >> 3) - 2;
    const int x_ = x + dx, y_ = y + dy;
    if (x_ < 0 || x_ > 8 || y_ < 0 || y_ > 9) continue;
    if (bit96(bb.own, y_ * 9 + x_)) continue;                // can_move
    if (c == PC_P) {
      if (y < 5 && x_ != x) continue;                        // no sideways step before the river
    } else if (c == PC_N || c == PC_E) {
      if (bit96(bb.occ, (y + dy / 2) * 9 + (x + dx / 2))) continue;   // leg / eye blocked
      if (c == PC_E && y_ > 4) continue;
    } else {
      if (x_ < 3 || x_ > 5) continue;
      if (y_ > 2) continue;
    }
    valid |= 1u << i;
  }
  pm->valid = valid;
  pm->count = czs::popc(valid) * (pm->fly >= 0 ? 2 : 1);
}
// writes the described moves, in the reference order, to list[pos ...]; entries past MAX_MOVES are dropped
CZ_D void piece_emit(const PieceMoves& pm, int from, move_t* list, int pos) {
  EmitSink out{list, pos, from};
  if (pm.kind == 1) {
    const int x = pm.x, y = pm.y;
    for (int x_ = pm.l + 1; x_ < x; ++x_) out(y * 9 + x_);
    for (int x_ = x + 1; x_ < pm.r; ++x_) out(y * 9 + x_);
    for (int y_ = pm.d + 1; y_ < y; ++y_) out(y_ * 9 + x);
    for (int y_ = y + 1; y_ < pm.u; ++y_) out(y_ * 9 + x);
    for (int k = 0; k < 4; ++k) if (pm.cap[k] >= 0) out(pm.cap[k]);
  } else if (pm.kind == 2) {
    for (int i = 0; i < pm.nd; ++i) {
      if (!((pm.valid >> i) & 1u)) continue;
      const int dd = (int)((pm.dirs >> (6 * i)) & 63);
      out((pm.y + (dd >> 3) - 2) * 9 + pm.x + (dd & 7) - 2);
      if (pm.fly >= 0) out(pm.fly);
    }
  }
}

// Ordered pseudo-legal move list of the side to move (static_env.py:256-321).
// The reference scans squares y-major then x (== ascending sq) and emits each piece's moves in turn.  Here the own
// pieces are compacted in that order (the `own` ballots), piece k goes to lane k % 32, describes its moves once from the
// bitboards, and one warp scan of the counts places every piece's block in the list.  Returns the count (<= MAX_MOVES).
CZ_DN int movegen(const uint8_t* b, move_t* list) {
  BoardBits bb;
  board_bits(b, &bb);
  const int n0 = czs::popc(bb.own[0]), n1 = czs::popc(bb.own[1]), n2 = czs::popc(bb.own[2]);
  const int pieces = n0 + n1 + n2;
  int base = 0;
  for (int first = 0; first < pieces; first += 32) {
    const int k = first + czs::lane();                       // this lane's piece, in scan order
    int sq = -1;
    if (k < n0) sq = czs::nth_set_bit(bb.own[0], k);
    else if (k < n0 + n1) sq = 32 + czs::nth_set_bit(bb.own[1], k - n0);
    else if (k < pieces) sq = 64 + czs::nth_set_bit(bb.own[2], k - n0 - n1);
    const uint8_t c = sq >= 0 ? b[sq] : (uint8_t)0;
    PieceMoves pm;
    piece_moves(b, bb, sq, c, &pm);
    int tot;
    const int off = czs::warp_excl_scan(pm.count, &tot);
    if (pm.count) piece_emit(pm, sq, list, base + off);
    base += tot;
  }
  czs::syncwarp();
  return base < MAX_MOVES ? base : MAX_MOVES;
}

// first index i < n with mv_to(list[i]) == target, or -1
CZ_D int first_move_to(const move_t* list, int n, int target) {
  int best = 0x7fffffff;
  for (int i = czs::lane(); i < n; i += 32)
    if (mv_to(list[i]) == target && i < best) best = i;
  for (int m = 16; m; m >>= 1) { int o = czs::shfl_xor(best, m); best = o < best ? o : best; }
  return best == 0x7fffffff ? -1 : best;
}

// square of the first piece with code `code` in scan order, or -1
CZ_D int find_piece_last(const uint8_t* b, uint8_t code) {
  // done() (static_env.py:25-32) keeps the LAST match of its scan; positions reached by play
  // have one king, arbitrary API input may not.
  int found = -1;
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    const unsigned m = czs::ballot(sq < NSQ && b[sq] == code);
    if (m) found = j * 32 + czs::fls(m) - 1;
  }
  return found;
}

// out = board after `m`, rotated 180 degrees with colours swapped (step + fliped_state,
// static_env.py:79-86,245-254).  in == out is allowed.  Returns no_eat (new_step :88-98).
CZ_D bool step_flip(const uint8_t* in, move_t m, uint8_t* out) {
  const int f = mv_from(m), t = mv_to(m);
  const bool no_eat = in[t] == 0;
  uint8_t v[3];
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    uint8_t c = 0;
    if (sq < NSQ) c = sq == t ? in[f] : (sq == f ? (uint8_t)0 : in[sq]);
    v[j] = c ? (uint8_t)(c ^ 8) : (uint8_t)0;
  }
  czs::syncwarp();
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    if (sq < NSQ) out[89 - sq] = v[j];
  }
  czs::syncwarp();
  return no_eat;
}

// fliped_state alone (static_env.py:245-254): the same position seen by the other side.
CZ_D void flip_only(const uint8_t* in, uint8_t* out) {
  uint8_t v[3];
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    const uint8_t c = sq < NSQ ? in[sq] : (uint8_t)0;
    v[j] = c ? (uint8_t)(c ^ 8) : (uint8_t)0;
  }
  czs::syncwarp();
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    if (sq < NSQ) out[89 - sq] = v[j];
  }
  czs::syncwarp();
}

// Left-right mirror across the central file (x -> 8 - x): square y*9+x goes to y*9+(8-x), the 6 pad bytes are copied.
// The rules are symmetric under it and boards are mover-relative, so it commutes with step_flip.  in == out is allowed.
CZ_D void mirror_board(const uint8_t* in, uint8_t* out) {
  uint8_t v[3];
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    v[j] = sq < BOARD_STRIDE ? in[sq] : (uint8_t)0;
  }
  czs::syncwarp();
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    if (sq < NSQ) out[sq + 8 - 2 * (sq % 9)] = v[j];
    else if (sq < BOARD_STRIDE) out[sq] = v[j];
  }
  czs::syncwarp();
}

CZ_D void copy_board(const uint8_t* in, uint8_t* out) {
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    if (sq < NSQ) out[sq] = in[sq];
  }
  czs::syncwarp();
}

// 128-bit position key: XOR over squares of two independent 64-bit mixes of (sq, code).
// The reference keys its tree by the canonical state string (player.py:49,211); two boards
// get the same key iff they are the same string (up to a 2^-128 collision).
CZ_HD uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
  return z ^ (z >> 31);
}
CZ_D void board_key(const uint8_t* b, uint64_t* k0, uint64_t* k1) {
  uint64_t a = 0, c = 0;
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    if (sq < NSQ && b[sq]) {
      const uint64_t t = (uint64_t)(sq * 16 + b[sq]);
      a ^= mix64(t + 0x9e3779b97f4a7c15ULL);
      c ^= mix64((t << 17) ^ 0xd1b54a32d192ed03ULL);
    }
  }
  *k0 = czs::warp_xor64(a);
  *k1 = czs::warp_xor64(c);
}

// ------------------------------------------------------------------ terminal test
struct DoneResult { int over; int v; int final_move; int check; };  // final_move = index into list or -1

// done() (static_env.py:14-77).  `list` receives the mover's move list when the position is
// not decided by king presence / facing kings (n_moves = -1 otherwise).  `sb`,`sl` are a
// scratch board / list used only for need_check.
CZ_D DoneResult done_eval(const uint8_t* b, move_t* list, int* n_moves, bool need_check,
                          uint8_t* sb, move_t* sl) {
  DoneResult r; r.over = 0; r.v = 0; r.final_move = -1; r.check = 0;
  *n_moves = -1;
  const int own_k = find_piece_last(b, PC_K);
  const int opp_k = find_piece_last(b, PC_K | PC_OPP);
  if (opp_k < 0) { r.over = 1; r.v = 1; return r; }      // 's' not in state
  if (own_k < 0) { r.over = 1; r.v = -1; return r; }     // 'S' not in state
  if (own_k == 0) { r.over = 1; r.v = -1; }              // the reference's (0,0) sentinel tests
  else if (opp_k == 0) { r.over = 1; r.v = 1; }
  else if (own_k % 9 == opp_k % 9) {
    const int x = own_k % 9, y0 = own_k / 9, y1 = opp_k / 9;
    const int y = y0 + 1 + czs::lane();
    const bool blocked = czs::any(y < y1 && b[y * 9 + x] != 0);
    if (!blocked) { r.over = 1; r.v = 1; }
  }
  if (!r.over) {
    const int n = movegen(b, list);
    *n_moves = n;
    const int i = first_move_to(list, n, opp_k);
    if (i >= 0) { r.over = 1; r.v = 1; r.final_move = i; }
  }
  if (!r.over && need_check) {
    flip_only(b, sb);
    const int n2 = movegen(sb, sl);
    r.check = first_move_to(sl, n2, 89 - own_k) >= 0 ? 1 : 0;
  }
  return r;
}

// has_attack_chessman (static_env.py:471-479): any rook / knight / pawn / cannon left.
CZ_D bool has_attack_chessman(const uint8_t* b) {
  bool p = false;
  for (int j = 0; j < 3; ++j) {
    const int sq = j * 32 + czs::lane();
    if (sq < NSQ) { const int t = b[sq] & 7; p = p || (b[sq] != 0 && (t == PC_R || t == PC_N || t == PC_P || t == PC_C)); }
  }
  return czs::any(p);
}

// ------------------------------------------------------------------ repetition helpers
struct EnvScratch {             // per-warp scratch in shared memory
  uint8_t b0[BOARD_STRIDE], b1[BOARD_STRIDE], b2[BOARD_STRIDE];
  move_t l0[MAX_MOVES], l1[MAX_MOVES], l2[MAX_MOVES];
  uint32_t s0[MAX_MOVES], s1[MAX_MOVES];
};

// be_catched (static_env.py:456-469): is the piece standing on mv_from(m) attacked right now.
CZ_DN bool be_catched(const uint8_t* b, move_t m, EnvScratch* sc) {
  flip_only(b, sc->b2);
  const int n = movegen(sc->b2, sc->l2);
  return first_move_to(sc->l2, n, 89 - mv_from(m)) >= 0;
}

// get_catch_list (static_env.py:423-454): set of (piece, from, target, to) the mover threatens
// to capture for free.  Keys are written to `set` (deduplicated); returns the set size.
CZ_DN int catch_list(const uint8_t* b, const move_t* moves, int n, uint32_t* set, EnvScratch* sc) {
  int cnt = 0;
  for (int i = 0; i < n; ++i) {
    const move_t m = moves[i];
    const int f = mv_from(m), t = mv_to(m);
    const uint8_t pf = b[f], pt = b[t];
    if (pt == 0) continue;                                   // not a capture
    step_flip(b, m, sc->b2);
    const int n2 = movegen(sc->b2, sc->l2);
    if (first_move_to(sc->l2, n2, 89 - t) >= 0) continue;    // can be recaptured
    if (pf == PC_P && f / 9 <= 4) continue;                  // pawn that has not crossed
    if (pt == (PC_P | PC_OPP) && t / 9 > 4) continue;        // their pawn on their own side
    if ((pf & 7) == (pt & 7)) continue;                      // an exchange
    const uint32_t key = (uint32_t)f | ((uint32_t)t << 7) | ((uint32_t)pf << 14) | ((uint32_t)pt << 18);
    bool dup = false;
    for (int k = czs::lane(); k < cnt; k += 32) dup = dup || set[k] == key;
    if (czs::any(dup)) continue;
    if (czs::lane() == 0) set[cnt] = key;
    ++cnt;
    czs::syncwarp();
  }
  return cnt;
}

// will_check_or_catch (static_env.py:390-421): does playing `m` give check or create a new
// unanswerable capture threat.
CZ_DN bool will_check_or_catch(const uint8_t* b, move_t m, EnvScratch* sc) {
  step_flip(b, m, sc->b0);                                   // state after the move (their view)
  const int their_k = find_piece_last(sc->b0, PC_K);
  flip_only(sc->b0, sc->b1);                                 // black_state: mover to move again
  const int n1 = movegen(sc->b1, sc->l1);
  // red_k defaults to [0,0] when absent (static_env.py:397-407) -> flipped square 89
  const int target = their_k < 0 ? 89 : 89 - their_k;
  if (first_move_to(sc->l1, n1, target) >= 0) return true;
  const int n0 = movegen(b, sc->l0);
  const int c0 = catch_list(b, sc->l0, n0, sc->s0, sc);
  const int c1 = catch_list(sc->b1, sc->l1, n1, sc->s1, sc);
  bool fresh = false;                                        // second_set - first_set != {}
  for (int k = czs::lane(); k < c1; k += 32) {
    bool in0 = false;
    for (int j = 0; j < c0; ++j) in0 = in0 || sc->s0[j] == sc->s1[k];
    fresh = fresh || !in0;
  }
  return czs::any(fresh) && c1 >= c0;
}

// ------------------------------------------------------------------ plane encoding
// state_to_planes (static_env.py:137-156): out[plane][row][col] f32, row = 9 - y.
CZ_D void encode_planes_f32(const uint8_t* b, float* out) {
  for (int i = czs::lane(); i < 14 * NSQ; i += 32) {
    const int pl = i / NSQ, r = (i % NSQ) / 9, x = i % 9;
    const uint8_t c = b[(9 - r) * 9 + x];
    const int p = c == 0 ? -1 : (pc_opp(c) ? c - 2 : c - 1);
    out[i] = p == pl ? 1.0f : 0.0f;
  }
}

}  // namespace cz
