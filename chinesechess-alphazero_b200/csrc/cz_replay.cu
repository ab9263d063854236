// cz_replay.cu — replay of human game records on the rules board, one warp per game (cz_sl_replay), and of the
// project's own self-play records (cz_play_replay, at the end of the file).
//
// Restates what the reference's supervised workers feed Keras: worker/sl.py load_game :124-174 (WXF moves resolved on the
// light board, light_env/chessboard.py parse_WXF_move :312-356 and find_row :358-398) and worker/sl_onegreen.py
// load_game :134-175 (static_env.py parse_onegreen_move :375-378).  The light board applies a move without checking it
// (push :256-259), so the replay applies exactly the move the reference would, legal or not; legality under the
// project's rules (movegen) is only reported.  Builds with nvcc (product) or g++ -DCZ_EMUL.
//
// The board is kept in the light board's own frame: sq = y*9 + x, y = 0 is red's back rank, red pieces (the light
// board's lower case) carry codes 1..7, black pieces 9..15.  The light board's side to move flips on every push,
// whatever list the move came from.  The observation of a ply (env.observation) is that board when red is to move and
// its flip_only otherwise: exactly the engine's mover-relative board.
#include "../../include/cczero_b200.h"
#include "cz_env.cuh"
#include "cz_rt.h"
#include "cz_err.h"

using namespace cz;

namespace {

constexpr int kWarpsPerBlock = 4;

struct ReplaySmem {
  uint8_t a[BOARD_STRIDE];      // the light board
  uint8_t obs[BOARD_STRIDE];    // the mover-relative observation
  move_t list[MAX_MOVES];
};

CZ_D ReplaySmem* my_smem() { return reinterpret_cast<ReplaySmem*>(czs::dyn_smem()) + czs::warp_in_block(); }

CZ_D bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }
CZ_D bool is_lower(uint8_t c) { return c >= 'a' && c <= 'z'; }
CZ_D bool is_upper(uint8_t c) { return c >= 'A' && c <= 'Z'; }

// board code of a light-board piece letter (lower case red), 0 for '.', -1 for a character no square holds
CZ_D int light_code(uint8_t c) {
  if (c == '.') return 0;
  const bool up = is_upper(c);
  const uint8_t l = up ? (uint8_t)(c + 32) : c;
  int t;
  switch (l) {
    case 'p': t = PC_P; break;
    case 'c': t = PC_C; break;
    case 'r': t = PC_R; break;
    case 'n': t = PC_N; break;
    case 'b': t = PC_E; break;
    case 'a': t = PC_A; break;
    case 'k': t = PC_K; break;
    default: return -1;
  }
  if (!up && !is_lower(c)) return -1;
  return up ? (t | PC_OPP) : t;
}

// str(v) appended to buf (v in -99..99)
CZ_D void append_int(char* buf, int* len, int v) {
  if (v < 0) { buf[(*len)++] = '-'; v = -v; }
  if (v >= 10) buf[(*len)++] = (char)('0' + v / 10);
  buf[(*len)++] = (char)('0' + v % 10);
}

struct Resolved {
  bool fail;          // the reference raises
  bool has_label;     // the move string is one of ActionLabelsRed
  int f, t;           // squares the light board's push reads and writes (valid unless fail)
  int lab_from, lab_to;
};

// move_to_str(src_col, src_row, dest_col, dest_row) handed to build_policy and Move(): the label exists for a 4-character
// string naming two on-board squares; Move() parses the first four characters and push() indexes the board with them.
CZ_D Resolved finish_move(int sc, int sr, int dc, int dr) {
  Resolved r; r.fail = false; r.has_label = false; r.f = r.t = 0; r.lab_from = r.lab_to = 0;
  char s[12]; int n = 0;
  append_int(s, &n, sc); append_int(s, &n, sr); append_int(s, &n, dc); append_int(s, &n, dr);
  if (n == 4 && sc <= 8 && dc <= 8) { r.has_label = true; r.lab_from = sr * 9 + sc; r.lab_to = dr * 9 + dc; }
  for (int i = 0; i < 4; ++i) if (!(s[i] >= '0' && s[i] <= '9')) { r.fail = true; return r; }    // int('-')
  const int x0 = s[0] - '0', y0 = s[1] - '0', x1 = s[2] - '0', y1 = s[3] - '0';
  if (x0 > 8 || x1 > 8) { r.fail = true; return r; }                                                // board[y][9]
  r.f = y0 * 9 + x0; r.t = y1 * 9 + x1;
  return r;
}

// parse_WXF_move + find_row on the light board `a`
CZ_D Resolved resolve_wxf(const uint8_t* a, const uint8_t* w) {
  Resolved bad; bad.fail = true; bad.has_label = false; bad.f = bad.t = bad.lab_from = bad.lab_to = 0;
  for (int i = 0; i < 4; ++i) if (w[i] == 0) return bad;                        // wxf[i]: IndexError
  uint8_t p = w[0];
  if (is_upper(p)) p = (uint8_t)(p + 32); else if (is_lower(p)) p = (uint8_t)(p - 32);   // swapcase
  const bool lower = is_lower(p), upper = is_upper(p);
  const uint8_t pl = lower ? p : (uint8_t)(p + 32);
  uint8_t fp = p;                                                                // find_row: h -> n, e -> b
  if (pl == 'h' && (lower || upper)) fp = lower ? 'n' : 'N';
  if (pl == 'e' && (lower || upper)) fp = lower ? 'b' : 'B';
  const int target = light_code(fp);
  const uint8_t col = w[1], mov = w[2], dch = w[3];
  int src_row = -1, src_col;
  if (is_digit(col)) {
    const int d = col - '0';
    src_col = upper ? 9 - d : d - 1;
    if (src_col == 9) return bad;                                                // board[i][9]
    const int scan = src_col < 0 ? 8 : src_col;                                  // board[i][-1] is column 8
    for (int i = 0; i < 10; ++i) if (target >= 0 && a[i * 9 + scan] == target) { src_row = i; break; }
  } else {
    // per column j (one lane each): how many squares hold the piece and the rows of the first two
    const int j = czs::lane();
    int cnt = 0, r1 = -1, r2 = -1;
    if (j < 9 && target >= 0)
      for (int i = 0; i < 10; ++i)
        if (a[i * 9 + j] == target) { if (cnt == 0) r1 = i; else if (cnt == 1) r2 = i; ++cnt; }
    int first = -1, second = -1, column = -1;
    for (int jj = 0; jj < 9; ++jj) {            // the reference's loop: `column` resets per file, first_row does not
      const int c = czs::shfl(cnt, jj), a1 = czs::shfl(r1, jj), a2 = czs::shfl(r2, jj);
      column = -1;
      if (c >= 1) { column = jj; first = a1; }
      if (c >= 2) { second = a2; break; }
    }
    src_col = column;
    src_row = ((lower && col == '+') || (upper && col == '-')) ? second : first;
  }
  int dest_col, dest_row;
  if (!is_digit(dch)) return bad;                                                // int(dest_col)
  const int d = dch - '0';
  const bool up_move = (mov == '+' && lower) || (mov == '-' && upper);
  if (mov == '.' || mov == '=') {
    dest_row = src_row;
    dest_col = lower ? d - 1 : 9 - d;
  } else if (pl == 'h' || pl == 'e' || pl == 'a') {                              // only letters reach these codes
    dest_col = lower ? d - 1 : 9 - d;
    int step;
    if (pl == 'h') step = (dest_col - src_col == 2 || src_col - dest_col == 2) ? 1 : 2;
    else if (pl == 'e') step = 2;
    else step = 1;
    dest_row = up_move ? src_row + step : src_row - step;
  } else {
    dest_row = up_move ? src_row + d : src_row - d;
    dest_col = src_col;
  }
  return finish_move(src_col, src_row, dest_col, dest_row);
}

// parse_onegreen_move: four digits "x0 y0 x1 y1" with y counted from black's side
CZ_D Resolved resolve_onegreen(const uint8_t* w) {
  Resolved bad; bad.fail = true; bad.has_label = false; bad.f = bad.t = bad.lab_from = bad.lab_to = 0;
  for (int i = 0; i < 4; ++i) if (!is_digit(w[i])) return bad;                  // int(move[i]) / IndexError
  return finish_move(w[0] - '0', 9 - (w[1] - '0'), w[2] - '0', 9 - (w[3] - '0'));
}

// static_env.evaluate piece values by engine code (P C R N E A K): state letters P C R K E M S
CZ_D int piece_value(int t) {
  switch (t) { case PC_P: return 1; case PC_C: return 5; case PC_R: return 14; case PC_N: return 7;
               case PC_E: return 3; case PC_A: return 2; case PC_K: return 1; default: return 0; }
}

CZ_KERNEL(k_sl_replay)(const uint8_t* init, const int32_t* offs, const uint8_t* plies, const int8_t* sides, int n, int mode,
                       const int16_t* lut, uint8_t* boards_out, int16_t* labels_out, int32_t* game_out) {
  const int g = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (g >= n) return;
  ReplaySmem* sm = my_smem();
  for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) { sm->a[k] = k < NSQ ? init[(size_t)g * BOARD_STRIDE + k] : 0; sm->obs[k] = 0; }
  czs::syncwarp();
  const int o0 = offs[g], o1 = offs[g + 1];
  bool red = true;                                   // the light board's turn
  int status = 0, done = 0, first_illegal = -1;
  for (int o = o0; o < o1; ++o) {
    const uint8_t* w = plies + (size_t)o * 4;
    const Resolved r = mode == CZ_SL_ONEGREEN ? resolve_onegreen(w) : resolve_wxf(sm->a, w);
    // the observation before the move, mover-relative
    if (red) copy_board(sm->a, sm->obs); else flip_only(sm->a, sm->obs);
    int lab = -1;
    if (r.has_label) {
      const bool black_list = sides[o] < 0;          // build_policy(action, flip=black): the label in the mover's frame
      lab = black_list ? lut[(89 - r.lab_from) * 90 + (89 - r.lab_to)] : lut[r.lab_from * 90 + r.lab_to];
    }
    if (mode == CZ_SL_ONEGREEN && lab < 0) { status = CZ_SL_FAILED; break; }       // build_policy raised: game dropped
    if (r.fail) { status = CZ_SL_FAILED; break; }
    // legality under the project's rules (diagnostic): the applied move in the mover's frame is in movegen's list
    const int nm = movegen(sm->obs, sm->list);
    const int mf = red ? r.f : 89 - r.f, mt = red ? r.t : 89 - r.t;
    const move_t want = mv_make(mf, mt);
    bool found = false;
    for (int i = czs::lane(); i < nm; i += 32) found = found || sm->list[i] == want;
    if (first_illegal < 0 && (lab < 0 || !czs::any(found))) first_illegal = o - o0;
    uint8_t* dst = boards_out + (size_t)o * BOARD_STRIDE;
    czs::syncwarp();
    if (czs::lane() < BOARD_STRIDE / 16) reinterpret_cast<uint4*>(dst)[czs::lane()] = reinterpret_cast<const uint4*>(sm->obs)[czs::lane()];
    if (czs::lane() == 0) {
      labels_out[o] = (int16_t)lab;
      const uint8_t pc = sm->a[r.f];                 // push: board[n] = board[p]; board[p] = '.'
      sm->a[r.t] = pc;
      sm->a[r.f] = 0;
    }
    czs::syncwarp();
    red = !red;
    ++done;
  }
  // static_env.evaluate(env.get_state()) on the final observation: upper case (the mover) counts +, lower case -
  if (red) copy_board(sm->a, sm->obs); else flip_only(sm->a, sm->obs);
  int ans = 0, tot = 0;
  for (int k = czs::lane(); k < NSQ; k += 32) {
    const uint8_t c = sm->obs[k];
    if (c) { const int v = piece_value(c & 7); tot += v; ans += pc_opp(c) ? -v : v; }
  }
  ans = czs::warp_sum(ans); tot = czs::warp_sum(tot);
  if (czs::lane() == 0) {
    int32_t* go = game_out + (size_t)g * CZ_SL_GAME_FIELDS;
    go[0] = done; go[1] = status; go[2] = first_illegal; go[3] = ans; go[4] = tot; go[5] = red ? 1 : 0;
  }
}

// Self-play records (cz_play_replay): the board is the engine's mover-relative board throughout, and a ply is exactly
// senv.step (static_env.py:79-86, step + fliped_state), i.e. step_flip, applied unchecked like records.expanding_data
// applies it through cz_env_step.
struct PlaySmem {
  uint8_t board[BOARD_STRIDE];
};

CZ_KERNEL(k_play_replay)(const uint8_t* init, const int32_t* offs, const uint16_t* moves, int n, const int16_t* lut,
                         uint8_t* boards_out, int16_t* labels_out, int32_t* status_out) {
  const int g = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (g >= n) return;
  uint8_t* b = (reinterpret_cast<PlaySmem*>(czs::dyn_smem()) + czs::warp_in_block())->board;
  for (int k = czs::lane(); k < BOARD_STRIDE; k += 32) b[k] = k < NSQ ? init[(size_t)g * BOARD_STRIDE + k] : 0;
  czs::syncwarp();
  const int o0 = offs[g], o1 = offs[g + 1];
  int status = CZ_PLAY_OK;
  for (int o = o0; o < o1; ++o) {
    const move_t m = moves[o];
    const bool on_board = mv_from(m) < NSQ && mv_to(m) < NSQ;
    const int lab = on_board ? lut[mv_from(m) * 90 + mv_to(m)] : -1;
    if (czs::lane() < BOARD_STRIDE / 16)
      reinterpret_cast<uint4*>(boards_out + (size_t)o * BOARD_STRIDE)[czs::lane()] = reinterpret_cast<const uint4*>(b)[czs::lane()];
    if (czs::lane() == 0) labels_out[o] = (int16_t)lab;
    if (lab < 0) { status = CZ_PLAY_FAILED; break; }       // expanding_data raises: "move ... is not an action label"
    step_flip(b, m, b);                                    // reads the board, syncs the warp, then writes it
  }
  if (czs::lane() == 0) status_out[g] = status;
}

// Training targets of visit-recorded plies (cz_visit_targets), one warp per row: target[l_i] = float32(n_i / sum n) with
// the sum in integers and the division in float64, i.e. numpy's `policy /= np.sum(policy)` on calc_policy's float64
// counts (player.py:375-406) followed by np.asarray(..., float32).  A row without pairs is the one-hot of its move.
CZ_KERNEL(k_visit_targets)(const int64_t* offs, const uint16_t* labels, const uint32_t* counts, const int16_t* move_labels,
                           const int64_t* ids, int n, float* out) {
  const int r = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (r >= n) return;
  const int64_t id = ids[r], o0 = offs[id], o1 = offs[id + 1];
  float* row = out + (size_t)r * N_LABELS;
  for (int k = czs::lane(); k < N_LABELS; k += 32) row[k] = 0.f;
  unsigned long long sum = 0;
  for (int64_t o = o0 + czs::lane(); o < o1; o += 32) sum += counts[o];
  for (int m = 16; m; m >>= 1) sum += czs::shfl_xor(sum, m);
  czs::syncwarp();
  if (o0 == o1) {
    if (czs::lane() == 0) row[move_labels[id]] = 1.f;
    return;
  }
#if defined(CZ_EMUL)
  const double den = (double)sum;
  for (int64_t o = o0 + czs::lane(); o < o1; o += 32) row[labels[o]] = (float)((double)counts[o] / den);
#else
  const double den = __ull2double_rn(sum);
  for (int64_t o = o0 + czs::lane(); o < o1; o += 32) row[labels[o]] = __double2float_rn(__ddiv_rn((double)counts[o], den));
#endif
}

}  // namespace

extern "C" {

int cz_visit_targets(const int64_t* offsets, const uint16_t* labels, const uint32_t* counts, const int16_t* move_labels,
                     const int64_t* ids, int n, float* out, void* stream) {
  if (n < 0) return cz_fail(CZ_ERR_ARG, "cz_visit_targets: bad n");
  if (n == 0) return CZ_OK;
  if (!offsets || !move_labels || !ids || !out) return cz_fail(CZ_ERR_ARG, "cz_visit_targets: null argument");
  CZ_LAUNCH(k_visit_targets, (n + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock, 0, (cz_stream_t)stream, offsets, labels,
            counts, move_labels, ids, n, out);
  const char* msg;
  const int e = czrt_last_error(&msg);
  if (e) return cz_fail(CZ_ERR_CUDA, "cz_visit_targets: %s", msg);
  return CZ_OK;
}

int cz_play_replay(const uint8_t* init_boards, const int32_t* ply_offsets, const uint16_t* moves, int n, const int16_t* lut,
                   uint8_t* boards_out, int16_t* labels_out, int32_t* status_out, void* stream) {
  if (n < 0) return cz_fail(CZ_ERR_ARG, "cz_play_replay: bad n");
  if (n == 0) return CZ_OK;
  if (!init_boards || !ply_offsets || !lut || !status_out) return cz_fail(CZ_ERR_ARG, "cz_play_replay: null argument");
  CZ_LAUNCH(k_play_replay, (n + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock, sizeof(PlaySmem) * kWarpsPerBlock,
            (cz_stream_t)stream, init_boards, ply_offsets, moves, n, lut, boards_out, labels_out, status_out);
  const char* msg;
  const int e = czrt_last_error(&msg);
  if (e) return cz_fail(CZ_ERR_CUDA, "cz_play_replay: %s", msg);
  return CZ_OK;
}

int cz_sl_replay(const uint8_t* init_boards, const int32_t* ply_offsets, const uint8_t* plies, const int8_t* sides, int n,
                 int mode, const int16_t* lut, uint8_t* boards_out, int16_t* labels_out, int32_t* game_out, void* stream) {
  if (n < 0 || (mode != CZ_SL_WXF && mode != CZ_SL_ONEGREEN)) return cz_fail(CZ_ERR_ARG, "cz_sl_replay: bad n or mode");
  if (n == 0) return CZ_OK;
  if (!init_boards || !ply_offsets || !lut || !game_out) return cz_fail(CZ_ERR_ARG, "cz_sl_replay: null argument");
  CZ_LAUNCH(k_sl_replay, (n + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock, sizeof(ReplaySmem) * kWarpsPerBlock,
            (cz_stream_t)stream, init_boards, ply_offsets, plies, sides, n, mode, lut, boards_out, labels_out, game_out);
  const char* msg;
  const int e = czrt_last_error(&msg);
  if (e) return cz_fail(CZ_ERR_CUDA, "cz_sl_replay: %s", msg);
  return CZ_OK;
}

}  // extern "C"
