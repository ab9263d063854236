// cz_env_api.cu — batched rules kernels (one warp per board) and their C-ABI entry points.
// Also holds the host-side action-label table.  Builds with nvcc (product) or g++ -DCZ_EMUL.
#include "../../include/cczero_b200.h"
#include "cz_env.cuh"
#include "cz_rt.h"
#include "cz_err.h"

using namespace cz;

namespace {

constexpr int kWarpsPerBlock = 4;

struct EnvWarpSmem {
  uint8_t board[BOARD_STRIDE];
  move_t list[MAX_MOVES];
  EnvScratch sc;
};

CZ_D EnvWarpSmem* my_smem() {
  return reinterpret_cast<EnvWarpSmem*>(czs::dyn_smem()) + czs::warp_in_block();
}

// 96-byte board, 16-byte aligned in global memory: lanes 0..5 move one uint4 each.
CZ_D void load_board(const uint8_t* g, uint8_t* s) {
  if (czs::lane() < BOARD_STRIDE / 16)
    reinterpret_cast<uint4*>(s)[czs::lane()] = czs::ldg(reinterpret_cast<const uint4*>(g) + czs::lane());
  czs::syncwarp();
}
CZ_D void store_board(const uint8_t* s, uint8_t* g) {
  czs::syncwarp();
  if (czs::lane() < BOARD_STRIDE / 16)
    reinterpret_cast<uint4*>(g)[czs::lane()] = reinterpret_cast<const uint4*>(s)[czs::lane()];
}

CZ_KERNEL(k_env_movegen)(const uint8_t* boards, int n, move_t* moves, int32_t* counts) {
  const int i = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (i >= n) return;
  EnvWarpSmem* sm = my_smem();
  load_board(boards + (size_t)i * BOARD_STRIDE, sm->board);
  const int cnt = movegen(sm->board, sm->list);
  for (int k = czs::lane(); k < MAX_MOVES; k += 32)
    moves[(size_t)i * MAX_MOVES + k] = k < cnt ? sm->list[k] : (move_t)0xFFFF;
  if (czs::lane() == 0) counts[i] = cnt;
}

CZ_KERNEL(k_env_done)(const uint8_t* boards, int n, int need_check, int8_t* out, uint16_t* final_move) {
  const int i = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (i >= n) return;
  EnvWarpSmem* sm = my_smem();
  load_board(boards + (size_t)i * BOARD_STRIDE, sm->board);
  int nm;
  const DoneResult r = done_eval(sm->board, sm->list, &nm, need_check != 0, sm->sc.b0, sm->sc.l0);
  if (czs::lane() == 0) {
    out[i * 4 + 0] = (int8_t)r.over;
    out[i * 4 + 1] = (int8_t)r.v;
    out[i * 4 + 2] = (int8_t)r.check;
    out[i * 4 + 3] = 0;
    final_move[i] = r.final_move >= 0 ? sm->list[r.final_move] : (uint16_t)0xFFFF;
  }
}

CZ_KERNEL(k_env_step)(const uint8_t* boards, const uint16_t* mv, int n, uint8_t* boards_out, uint8_t* no_eat) {
  const int i = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (i >= n) return;
  EnvWarpSmem* sm = my_smem();
  load_board(boards + (size_t)i * BOARD_STRIDE, sm->board);
  for (int k = NSQ + czs::lane(); k < BOARD_STRIDE; k += 32) sm->sc.b0[k] = 0;
  const bool ne = step_flip(sm->board, mv[i], sm->sc.b0);
  store_board(sm->sc.b0, boards_out + (size_t)i * BOARD_STRIDE);
  if (no_eat && czs::lane() == 0) no_eat[i] = ne ? 1 : 0;
}

CZ_KERNEL(k_env_planes)(const uint8_t* boards, int n, float* planes) {
  const int i = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (i >= n) return;
  EnvWarpSmem* sm = my_smem();
  load_board(boards + (size_t)i * BOARD_STRIDE, sm->board);
  encode_planes_f32(sm->board, planes + (size_t)i * 14 * NSQ);
}

CZ_KERNEL(k_env_check_catch)(const uint8_t* boards, const uint16_t* mv, int n, uint8_t* wcc, uint8_t* bc, uint8_t* ha) {
  const int i = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (i >= n) return;
  EnvWarpSmem* sm = my_smem();
  load_board(boards + (size_t)i * BOARD_STRIDE, sm->board);
  if (wcc) { const bool r = will_check_or_catch(sm->board, mv[i], &sm->sc); if (czs::lane() == 0) wcc[i] = r; }
  if (bc) { const bool r = be_catched(sm->board, mv[i], &sm->sc); if (czs::lane() == 0) bc[i] = r; }
  if (ha) { const bool r = has_attack_chessman(sm->board); if (czs::lane() == 0) ha[i] = r; }
}

CZ_KERNEL(k_env_keys)(const uint8_t* boards, int n, uint64_t* keys) {
  const int i = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (i >= n) return;
  EnvWarpSmem* sm = my_smem();
  load_board(boards + (size_t)i * BOARD_STRIDE, sm->board);
  uint64_t k0, k1;
  board_key(sm->board, &k0, &k1);
  if (czs::lane() == 0) { keys[2 * i] = k0; keys[2 * i + 1] = k1; }
}

// flags NULL: every row mirrored; otherwise row i is mirrored where flags[i] != 0 and copied where it is 0.
CZ_KERNEL(k_env_mirror)(const uint8_t* boards, const uint8_t* flags, int n, uint8_t* out) {
  const int i = czs::block_idx() * czs::warps_per_block() + czs::warp_in_block();
  if (i >= n) return;
  EnvWarpSmem* sm = my_smem();
  load_board(boards + (size_t)i * BOARD_STRIDE, sm->board);
  if (!flags || flags[i]) mirror_board(sm->board, sm->board);
  store_board(sm->board, out + (size_t)i * BOARD_STRIDE);
}

int finish_launch(const char* what) {
  const char* msg;
  const int e = czrt_last_error(&msg);
  if (e) return cz_fail(CZ_ERR_CUDA, "%s: %s", what, msg);
  return CZ_OK;
}

}  // namespace

#define CZ_ENV_LAUNCH(kern, n, stream, ...) \
  CZ_LAUNCH(kern, ((n) + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock, sizeof(EnvWarpSmem) * kWarpsPerBlock, stream, __VA_ARGS__)

extern "C" {

int cz_env_movegen(const uint8_t* boards, int n, uint16_t* moves, int32_t* counts, void* stream) {
  if (n < 0 || (n && (!boards || !moves || !counts))) return cz_fail(CZ_ERR_ARG, "cz_env_movegen: bad argument");
  if (n == 0) return CZ_OK;
  CZ_ENV_LAUNCH(k_env_movegen, n, (cz_stream_t)stream, boards, n, moves, counts);
  return finish_launch("cz_env_movegen");
}

int cz_env_done(const uint8_t* boards, int n, int need_check, int8_t* out, uint16_t* final_move, void* stream) {
  if (n < 0 || (n && (!boards || !out || !final_move))) return cz_fail(CZ_ERR_ARG, "cz_env_done: bad argument");
  if (n == 0) return CZ_OK;
  CZ_ENV_LAUNCH(k_env_done, n, (cz_stream_t)stream, boards, n, need_check, out, final_move);
  return finish_launch("cz_env_done");
}

int cz_env_step(const uint8_t* boards, const uint16_t* moves, int n, uint8_t* boards_out, uint8_t* no_eat, void* stream) {
  if (n < 0 || (n && (!boards || !moves || !boards_out))) return cz_fail(CZ_ERR_ARG, "cz_env_step: bad argument");
  if (n == 0) return CZ_OK;
  CZ_ENV_LAUNCH(k_env_step, n, (cz_stream_t)stream, boards, moves, n, boards_out, no_eat);
  return finish_launch("cz_env_step");
}

int cz_env_encode_planes(const uint8_t* boards, int n, float* planes, void* stream) {
  if (n < 0 || (n && (!boards || !planes))) return cz_fail(CZ_ERR_ARG, "cz_env_encode_planes: bad argument");
  if (n == 0) return CZ_OK;
  CZ_ENV_LAUNCH(k_env_planes, n, (cz_stream_t)stream, boards, n, planes);
  return finish_launch("cz_env_encode_planes");
}

int cz_env_check_catch(const uint8_t* boards, const uint16_t* moves, int n, uint8_t* wcc, uint8_t* bc, uint8_t* ha,
                       void* stream) {
  if (n < 0 || (n && (!boards || ((wcc || bc) && !moves)))) return cz_fail(CZ_ERR_ARG, "cz_env_check_catch: bad argument");
  if (n == 0) return CZ_OK;
  CZ_ENV_LAUNCH(k_env_check_catch, n, (cz_stream_t)stream, boards, moves, n, wcc, bc, ha);
  return finish_launch("cz_env_check_catch");
}

int cz_env_keys(const uint8_t* boards, int n, uint64_t* keys, void* stream) {
  if (n < 0 || (n && (!boards || !keys))) return cz_fail(CZ_ERR_ARG, "cz_env_keys: bad argument");
  if (n == 0) return CZ_OK;
  CZ_ENV_LAUNCH(k_env_keys, n, (cz_stream_t)stream, boards, n, keys);
  return finish_launch("cz_env_keys");
}

int cz_env_mirror(const uint8_t* boards, const uint8_t* flags, int n, uint8_t* out, void* stream) {
  if (n < 0 || (n && (!boards || !out))) return cz_fail(CZ_ERR_ARG, "cz_env_mirror: bad argument");
  if (n == 0) return CZ_OK;
  CZ_ENV_LAUNCH(k_env_mirror, n, (cz_stream_t)stream, boards, flags, n, out);
  return finish_launch("cz_env_mirror");
}

// create_action_labels (environment/lookup_tables.py:62-132): per source square the same-row,
// same-column and knight-jump destinations, then the fixed advisor and elephant moves.
int cz_action_labels(char* labels, int16_t* lut) {
  if (!labels && !lut) return cz_fail(CZ_ERR_ARG, "cz_action_labels: both outputs NULL");
  int cnt = 0;
  if (lut) for (int i = 0; i < 8100; ++i) lut[i] = -1;
  auto add = [&](int x0, int y0, int x1, int y1) {
    if (cnt < CZ_N_LABELS) {
      if (labels) {
        labels[cnt * 4 + 0] = (char)('0' + x0); labels[cnt * 4 + 1] = (char)('0' + y0);
        labels[cnt * 4 + 2] = (char)('0' + x1); labels[cnt * 4 + 3] = (char)('0' + y1);
      }
      if (lut) lut[(y0 * 9 + x0) * 90 + (y1 * 9 + x1)] = (int16_t)cnt;
    }
    ++cnt;
  };
  static const int jumps[8][2] = {{-2, -1}, {-1, -2}, {-2, 1}, {1, -2}, {2, -1}, {-1, 2}, {2, 1}, {1, 2}};  // (dy, dx)
  for (int n1 = 0; n1 < 10; ++n1)
    for (int l1 = 0; l1 < 9; ++l1) {
      for (int t = 0; t < 9; ++t) if (t != l1) add(l1, n1, t, n1);
      for (int t = 0; t < 10; ++t) if (t != n1) add(l1, n1, l1, t);
      for (int j = 0; j < 8; ++j) {
        const int n2 = n1 + jumps[j][0], l2 = l1 + jumps[j][1];
        if (n2 >= 0 && n2 < 10 && l2 >= 0 && l2 < 9) add(l1, n1, l2, n2);
      }
    }
  static const char* fixed[] = {
      "3041", "5041", "3241", "5241", "4130", "4150", "4132", "4152",   // red advisors
      "3948", "5948", "3748", "5748", "4839", "4859", "4837", "4857",   // black advisors
      "2002", "2042", "6042", "6082", "2402", "2442", "6442", "6482",   // red elephants
      "0220", "4220", "4260", "8260", "0224", "4224", "4264", "8264",
      "2907", "2947", "6947", "6987", "2507", "2547", "6547", "6587",   // black elephants
      "0729", "4729", "4769", "8769", "0725", "4725", "4765", "8765"};
  for (const char* s : fixed) add(s[0] - '0', s[1] - '0', s[2] - '0', s[3] - '0');
  if (cnt != CZ_N_LABELS) return cz_fail(CZ_ERR_STATE, "cz_action_labels: built %d labels", cnt);
  return CZ_OK;
}

// M[l] = label of l's move reflected across the central file, built from cz_action_labels' strings and table.
int cz_mirror_labels(int16_t* m) {
  if (!m) return cz_fail(CZ_ERR_ARG, "cz_mirror_labels: NULL output");
  char labels[CZ_N_LABELS * 4];
  int16_t lut[8100];
  const int rc = cz_action_labels(labels, lut);
  if (rc) return rc;
  for (int l = 0; l < CZ_N_LABELS; ++l) {
    const char* s = labels + l * 4;
    const int x0 = 8 - (s[0] - '0'), y0 = s[1] - '0', x1 = 8 - (s[2] - '0'), y1 = s[3] - '0';
    m[l] = lut[(y0 * 9 + x0) * 90 + (y1 * 9 + x1)];
    if (m[l] < 0) return cz_fail(CZ_ERR_STATE, "cz_mirror_labels: label %d has no mirror", l);
  }
  return CZ_OK;
}

}  // extern "C"
