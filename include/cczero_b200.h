/* cczero_b200.h — C-ABI of libcczero_b200.so, the H100-native Xiangqi self-play hot path.
 *
 * The reference (NeymarL/ChineseChess-AlphaZero) is pure Python and has no FFI; the hot path
 * sits behind three Python surfaces (SURVEY.md §8b).  This header is what a ctypes binding of
 * those surfaces calls instead.  Each entry point cites the reference code it replaces
 * (paths relative to the reference root).
 *
 * Conventions
 *   - every function returns 0 on success or a negative cz_status; nothing throws across the ABI;
 *     cz_last_error() gives the message of the last failure on the calling thread.
 *   - "dev" pointers are device memory owned by the caller (torch CUDA tensors: .data_ptr());
 *     "host" pointers are ordinary host memory.  The library never frees caller memory.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream).  Calls are
 *     stream-ordered; only the functions documented as synchronising wait for the device.
 *   - boards: BOARD_STRIDE (96) bytes each, first 90 = squares sq = y*9+x with y = 0 the
 *     side-to-move's back rank; 0 empty, 1..7 = side-to-move P C R N E A K, 9..15 = opponent.
 *   - moves: uint16 (from << 8) | to.
 *   - one engine per GPU per process, driven by one host thread.
 */
#ifndef CCZERO_B200_H
#define CCZERO_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define CZ_BOARD_STRIDE 96
#define CZ_MAX_MOVES 128
#define CZ_N_LABELS 2086
#define CZ_MAX_NO_ACT 16

typedef enum cz_status {
  CZ_OK = 0,
  CZ_ERR_ARG = -1,        /* bad argument */
  CZ_ERR_CUDA = -2,       /* a CUDA runtime / driver call failed */
  CZ_ERR_STATE = -3,      /* call not valid in the engine's current state */
  CZ_ERR_CAPACITY = -4,   /* a fixed-capacity device pool overflowed */
  CZ_ERR_UNSUPPORTED = -5 /* e.g. tensor-core path requested in a build without it */
} cz_status;

const char* cz_last_error(void);
/* 1 when this build runs kernels on a CUDA device, 0 for the CPU SIMT-emulation test build
 * (tests/simt_emul; never shipped). */
int cz_build_is_cuda(void);

/* ------------------------------------------------------------------------------------------
 * Lookup tables — environment/lookup_tables.py:62-134 (create_action_labels / ActionLabelsRed)
 * labels_host: 2086*4 chars "x0y0x1y1" (no terminators); lut_host: 90*90 int16, label index of
 * (from,to) or -1.  Host-only, no device work.
 * ---------------------------------------------------------------------------------------- */
int cz_action_labels(char* labels_host, int16_t* lut_host);
/* Left-right mirror of the action labels (x -> 8 - x on both squares; the rules are symmetric across the central file):
 * lut_host [2086] int16, lut_host[l] = label of l's reflected move.  An involution whose 90 fixed points are the moves
 * along file 4.  Built from cz_action_labels.  Host-only, no device work. */
int cz_mirror_labels(int16_t* lut_host);

/* ------------------------------------------------------------------------------------------
 * Batched rules kernels (one warp per board) — environment/static_env.py
 * ---------------------------------------------------------------------------------------- */
/* get_legal_moves :256-321.  moves_dev [n][CZ_MAX_MOVES] in reference order, counts_dev [n]. */
int cz_env_movegen(const uint8_t* boards_dev, int n, uint16_t* moves_dev, int32_t* counts_dev, void* stream);
/* done :14-77.  out_dev [n][4] int8 = {over, v, check, 0}; final_move_dev [n] (0xFFFF = None). */
int cz_env_done(const uint8_t* boards_dev, int n, int need_check, int8_t* out_dev, uint16_t* final_move_dev,
                void* stream);
/* step / new_step :79-98 (move, then rotate + swap colours).  no_eat_dev may be NULL. */
int cz_env_step(const uint8_t* boards_dev, const uint16_t* moves_dev, int n, uint8_t* boards_out_dev,
                uint8_t* no_eat_dev, void* stream);
/* state_to_planes :137-156.  planes_dev [n][14][10][9] float32. */
int cz_env_encode_planes(const uint8_t* boards_dev, int n, float* planes_dev, void* stream);
/* will_check_or_catch :390-421, be_catched :456-469, has_attack_chessman :471-479.
 * Any of the three outputs may be NULL. */
int cz_env_check_catch(const uint8_t* boards_dev, const uint16_t* moves_dev, int n, uint8_t* will_cc_dev,
                       uint8_t* be_catched_dev, uint8_t* has_attack_dev, void* stream);
/* 128-bit canonical position keys (replaces the state-string dict key, agent/player.py:49). */
int cz_env_keys(const uint8_t* boards_dev, int n, uint64_t* keys_dev /* [n][2] */, void* stream);
/* Left-right mirror of boards [n][CZ_BOARD_STRIDE]: square y*9+x -> y*9+(8-x), pad bytes copied.  flags_dev [n] may be
 * NULL (every row mirrored); otherwise a row is mirrored where its flag is nonzero and copied unchanged where it is 0.
 * boards_dev == out_dev is allowed.  Pairs with cz_mirror_labels: movegen(mirror(b)) = cz_mirror_labels(movegen(b)). */
int cz_env_mirror(const uint8_t* boards_dev, const uint8_t* flags_dev, int n, uint8_t* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Human game records — worker/sl.py load_game :124-174 and worker/sl_onegreen.py load_game :134-175, one warp per game
 * ---------------------------------------------------------------------------------------- */
enum { CZ_SL_WXF = 0, CZ_SL_ONEGREEN = 1 };
enum { CZ_SL_OK = 0, CZ_SL_FAILED = 1 };   /* FAILED: the reference raises on this game, or (onegreen) drops it */
enum { CZ_SL_GAME_FIELDS = 6 };
/* Replays n games on the light board of the reference.  init_boards_dev [n][96]: the start position in the light board's
 * frame (y = 0 red's back rank, red pieces codes 1..7, black 9..15).  ply_offsets_dev [n + 1]: game g owns plies
 * [off[g], off[g+1]).  plies_dev [P][4]: the WXF characters ("C2.5", "H8+7", "R+.1"; missing characters 0) or the four
 * onegreen digits.  sides_dev [P]: +1 for a move of the red list, -1 for the black list (build_policy's flip).
 * lut_dev [90*90]: cz_action_labels' table.  Outputs per ply: boards_out_dev [P][96] the mover-relative observation
 * before the move (engine layout), labels_out_dev [P] the label in the mover's frame or -1 where the move has none.
 * game_out_dev [n][CZ_SL_GAME_FIELDS] int32 = {plies applied, status, first ply not in movegen's list or -1,
 * evaluate's ans and tot on the final observation, 1 if red is to move at the end}.  Plies after a failure are not
 * written. */
int cz_sl_replay(const uint8_t* init_boards_dev, const int32_t* ply_offsets_dev, const uint8_t* plies_dev,
                 const int8_t* sides_dev, int n, int mode, const int16_t* lut_dev, uint8_t* boards_out_dev,
                 int16_t* labels_out_dev, int32_t* game_out_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Self-play records — worker/optimize.py expanding_data :234-281 on the files worker/self_play.py :202-208 writes, one
 * warp per game
 * ---------------------------------------------------------------------------------------- */
enum { CZ_PLAY_OK = 0, CZ_PLAY_FAILED = 1 };   /* FAILED: a ply whose move has no action label (the reference raises) */
/* Replays n games of the reference's record format: an initial state, then moves "x0y0x1y1" in the mover's own frame.
 * init_boards_dev [n][96]: the initial state in engine layout (env.state_to_board).  ply_offsets_dev [n + 1]: game g owns
 * plies [off[g], off[g+1]).  moves_dev [P]: (from << 8) | to, squares y*9+x of the mover's frame.  lut_dev [90*90]:
 * cz_action_labels' table.  Each ply is senv.step (step_flip), applied unchecked.  Outputs per ply: boards_out_dev [P][96]
 * the mover-relative board before the move, labels_out_dev [P] the move's label or -1.  status_out_dev [n]: CZ_PLAY_OK,
 * or CZ_PLAY_FAILED at the first ply without a label (that ply's board and -1 are written, later plies are not). */
int cz_play_replay(const uint8_t* init_boards_dev, const int32_t* ply_offsets_dev, const uint16_t* moves_dev, int n,
                   const int16_t* lut_dev, uint8_t* boards_out_dev, int16_t* labels_out_dev, int32_t* status_out_dev,
                   void* stream);
/* Policy targets of n positions of a dataset whose plies carry root visit counts (cz_config.record_visits records): the
 * pairs of position p are offsets_dev[p] .. offsets_dev[p+1]-1 of labels_dev (u16, < 2086) / counts_dev (u32, > 0).
 * out_dev [n][2086] f32, row r for position ids_dev[r]: target[label] = float32(N / sum N), the sum in integers and the
 * division in float64 — numpy's `policy /= np.sum(policy)` on calc_policy's float64 counts (agent/player.py:403) then
 * np.asarray(..., float32).  A position without pairs gets the one-hot of move_labels_dev[p] (the reference's
 * build_policy(final_move), worker/self_play.py:180).  Stream-ordered. */
int cz_visit_targets(const int64_t* offsets_dev, const uint16_t* labels_dev, const uint32_t* counts_dev,
                     const int16_t* move_labels_dev, const int64_t* ids_dev, int n, float* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Search engine — agent/player.py (CChessPlayer) for many concurrent games
 * ---------------------------------------------------------------------------------------- */
typedef struct cz_engine cz_engine;

typedef struct cz_config {
  int32_t struct_bytes;        /* sizeof(cz_config), for ABI checking */
  int32_t device;              /* CUDA device ordinal */
  int32_t n_games;             /* concurrent games held by this engine */
  int32_t sims_per_move;       /* play_config.simulation_num_per_move */
  int32_t leaves_per_round;    /* config.play.search_threads (K): sims launched per round */
  int32_t virtual_loss;        /* config.play.virtual_loss */
  int32_t max_nodes_per_game;  /* node pool capacity per game */
  int32_t max_edges_per_game;  /* edge pool capacity per game */
  int32_t max_path;            /* longest root->leaf path stored per simulation */
  int32_t noise_mode;          /* 0 = host table (parity), 1 = on-device Philox gamma sampler: stream = (seed, rank, game slot,
                                * search number on that slot since the last reset), counter = draw index — every root visit of
                                * every move draws fresh noise like player.py:303-304 */
  int32_t max_plies;           /* 2*max_game_length, capacity of the per-game record */
  int32_t nn_filters;          /* cnn_filter_num (0 = no network, external evaluator only) */
  int32_t nn_blocks;           /* res_layer_num */
  int32_t nn_value_fc;         /* value_fc_size */
  double c_puct;               /* play_config.c_puct */
  double noise_eps;            /* play_config.noise_eps */
  double dirichlet_alpha;      /* play_config.dirichlet_alpha */
  double tau_decay_rate;       /* play_config.tau_decay_rate */
  double resign_threshold;     /* play_config.resign_threshold */
  double enable_resign_rate;   /* play_config.enable_resign_rate (self_play.py:102-105) */
  int32_t min_resign_turn;     /* play_config.min_resign_turn */
  int32_t max_game_length;     /* play_config.max_game_length */
  uint64_t seed;               /* Philox key (seed, rank) for the on-device streams */
  int32_t rank;                /* data-parallel rank, selects the RNG sub-stream */
  int32_t arena;               /* 1: evaluator arena (worker/evaluator.py:147-250): n_games = 2*M slots for M games; slot i holds
                                * player 0's tree of game i, slot i+M player 1's; player p is evaluated by network p
                                * (cz_nn_set_weights_net); the red side alternates with the game index; evaluator draw rules */
  int32_t nn_fp32_skip;        /* residual (skip) stream precision: 0 auto (fp32 when nn_blocks >= 10), 1 fp32, 2 fp16.
                                * fp32 keeps the value error of 20-block nets <= 6e-4 (fp16: up to 1.5e-3) for ~10 % time */
  int32_t use_history;         /* CChessPlayer(use_history=True) (player.py:45,326-334): 28 input planes, planes 14-27 = the
                                * position two plies earlier (static_env.py:158-194); leaf records become (board, history board) */
  int32_t game_quota;          /* > 0: the on-device game loop plays exactly the games with running index < game_quota (the
                                * `for idx in range(game_num)` of evaluator.py:104 / a bounded self-play run): a slot whose next
                                * game index would reach the quota retires instead of restarting.  0 = restart for ever */
  int32_t playouts_lo;         /* arena, > 0: every game draws its own simulations per move = randint(playouts_lo, playouts_hi) * 100 */
  int32_t playouts_hi;         /*   when it starts (evaluator.py:153-154: randint(8, 12) * 100), from the Philox stream of the game */
  int32_t nn_policy_channels;  /* filters of the policy 1x1 convolution: 0 = 4 (agent/model.py:47); the older shipped configs use 2
                                * (data/model/model_128f.json, model_256f.json) and 32 (model_128_l1_config.json) */
  int32_t nn_value_channels;   /* filters of the value 1x1 convolution: 0 = 2 (agent/model.py:56); the older configs use 4 */
  int32_t record_visits;       /* 1: the on-device game loop records every ply's root visit counts, calc_policy's N(s,a) with the
                                * no_act moves zeroed (agent/player.py:375-406; worker/self_play.py:112,134 keep the policy the
                                * reference commented out).  Read them with cz_drain_records_visits.  Not with arena */
  int32_t eval_mirror;         /* 1: every evaluation by the engine's own network in the device-driven loop (cz_search,
                                * cz_search_run, cz_play_move / cz_selfplay, the arena with each range's network) averages the
                                * leaf b and its left-right mirror Mb (cz_env_mirror):  p(l) = 0.5 * (pi(b)[l] + pi(Mb)[M l]),
                                * v = 0.5 * (v(b) + v(Mb)), M = cz_mirror_labels, each sum and product rounded once in fp32.  History
                                * engines mirror both boards of the leaf record.  Costs a second tower pass per leaf: the network's
                                * batch is 2 * n_games * leaves_per_round.  The host-driven calls (cz_search_wave, cz_leaf_*,
                                * cz_search_apply*) and cz_nn_forward* are unchanged: they apply what the caller hands them.
                                * Rejected without a network of the engine's own (nn_filters == 0) */
} cz_config;

/* Device workspace the caller must provide (a torch.uint8 CUDA tensor). */
int cz_workspace_bytes(const cz_config* cfg, uint64_t* bytes);
int cz_create(const cz_config* cfg, void* workspace_dev, uint64_t workspace_bytes, void* stream, cz_engine** out);
void cz_destroy(cz_engine* e);

/* Start games: boards_host [n_games][CZ_BOARD_STRIDE] or NULL for INIT_STATE (static_env.py:9).
 * Clears every tree (a new CChessPlayer with search_tree=None, player.py:48-51). */
int cz_reset_games(cz_engine* e, const uint8_t* boards_host);
/* Replace the root position of one game, keeping its tree (the per-move path of
 * worker/self_play.py:122-147: the same player object searches the next state). */
int cz_set_root(cz_engine* e, int game, const uint8_t* board_host);

/* Bulk variants for all games (host buffers [n_games][CZ_BOARD_STRIDE]; pinned memory makes them async):
 * cz_set_roots is stream-ordered, cz_get_roots synchronises. */
int cz_set_roots(cz_engine* e, const uint8_t* boards_host);
int cz_get_roots(cz_engine* e, uint8_t* boards_host);

typedef struct cz_root_opts {
  int32_t struct_bytes;            /* sizeof(cz_root_opts): checked like cz_config.struct_bytes */
  int32_t reserved;
  /* per game, may be NULL for "none" */
  const uint16_t* no_act_host;     /* [n_games][CZ_MAX_NO_ACT] moves banned at the root, 0xFFFF-terminated */
  const uint8_t* increase_temp_host; /* [n_games] */
  const uint8_t* active_host;      /* [n_games] 0 = skip this game */
  const double* noise_dev;         /* noise_mode 0: [n_games][noise_stride] Dirichlet[0] draws in call order */
  int64_t noise_stride;
  int32_t sims_override;           /* >0: depth argument of action() (player.py:160-161) */
  int32_t raw_tasks;               /* 1: run exactly sims_override simulations; the caller did the bookkeeping of
                                    * player.py:153-165 (done / depth / infinite) itself (UCI front end) */
  /* use_history engines: the `hist` argument of action() (player.py:150-151,215-216).  root_hist_given_host [n_games]:
   * 1 = a non-empty hist list was passed; root_hist_host [n_games][CZ_BOARD_STRIDE]: the position hist[-5] (all squares
   * empty when the list holds fewer than 5 entries).  Both NULL = no hist (worker/self_play.py:124 never passes one). */
  const uint8_t* root_hist_host;
  const uint8_t* root_hist_given_host;
} cz_root_opts;

/* CChessPlayer.action up to the search (player.py:145-186), split so that an external
 * evaluator can stand in for CChessModelAPI:
 *   cz_search_begin            tree reuse + task count (player.py:147-171)
 *   loop: cz_search_wave       descents until every queued simulation is at a leaf / terminal /
 *                              repetition / parked (MCTS_search, player.py:198-260), immediate
 *                              results backed up (update_tree, :340-373); returns #leaves to
 *                              evaluate and whether any game still has work (synchronises)
 *         cz_leaf_planes       state_to_planes of those leaves (expand_and_evaluate, :322-338)
 *         cz_search_apply      attach (policy, value) to the leaves, back up, resume parked sims
 * The schedule is the canonical one of SURVEY.md Appendix C. */
/* opts == NULL keeps the per-game options the on-device game loop maintains (no_act / increase_temp). */
int cz_search_begin(cz_engine* e, const cz_root_opts* opts);
int cz_search_wave(cz_engine* e, int32_t* n_leaves, int32_t* any_active);
int cz_leaf_planes(cz_engine* e, float* planes_dev /* [n_leaves][14][10][9]; [n_leaves][28][10][9] with use_history */);
int cz_leaf_boards(cz_engine* e, uint8_t* boards_dev /* [n_leaves][CZ_BOARD_STRIDE]; [n_leaves][2][CZ_BOARD_STRIDE] with use_history */);
int cz_search_apply(cz_engine* e, const float* policy_dev /* [n_leaves][2086] */, const float* value_dev /* [n_leaves] */);
/* The same hand-over without the 2086-vector: select_action_q_and_u (player.py:272-284) reads the policy only at the labels of
 * the leaf's legal moves, so an evaluator that is given those labels can return just those entries.
 *   cz_leaf_labels         labels_dev [n_leaves][CZ_MAX_MOVES] int16 = action label of each legal move in move-list order
 *                          (-1: the move has no label), counts_dev [n_leaves] int32
 *   cz_search_apply_legal  legal_p_dev [n_leaves][CZ_MAX_MOVES] f32 = policy[label] per legal move; everything downstream
 *                          (sequential f32 renormalisation, backup) is the code path of cz_search_apply
 * This is what the integrated search (cz_search) does on the device: the [n][2086] f32 row never exists there. */
int cz_leaf_labels(cz_engine* e, int16_t* labels_dev, int32_t* counts_dev);
int cz_search_apply_legal(cz_engine* e, const float* legal_p_dev, const float* value_dev);
/* n_sims more simulations for every active game inside the search cz_search_begin opened: same root options, the noise
 * table continues where it stopped, sims_run / noise_used keep counting.  Follow with the wave / apply loop.  Lets a host
 * loop run action()'s rounds (player.py:167-184) in slices: `go infinite` / movetime stops, `info depth` lines between. */
int cz_search_more(cz_engine* e, int32_t n_sims);
/* Replace the Dirichlet table of the open search (noise_mode 0) by a longer one holding the same draws plus more; the
 * per-game read position is kept.  Stream-ordered. */
int cz_set_noise_table(cz_engine* e, const double* noise_dev, int64_t noise_stride);
/* Whole search with the built-in network as evaluator (needs cz_nn_set_weights).  Device-driven: every wave / evaluation /
 * apply iteration is a fixed-shape sequence of launches whose batch size is a device integer, captured as a CUDA graph.  A
 * search is one launch of a graph whose WHILE node repeats the iteration until no game has work left.  The engine's first
 * search runs one iteration as plain launches, captures the graph and launches it for the rest; so does the first search
 * with cz_nn_profile on, which has a graph of its own (the same iteration with the tower bracketed by two timestamp kernels).
 * Synchronises once, at the end. */
int cz_search(cz_engine* e, const cz_root_opts* opts);
/* The loop of cz_search alone: run the simulations cz_search_begin / cz_search_more queued, built-in network as evaluator.
 * (A UCI front end slices action()'s rounds with cz_search_more and prints `info depth` lines in between.)  Synchronises. */
int cz_search_run(cz_engine* e);

typedef struct cz_root_info {
  int32_t n_moves;                 /* legal moves of the root (0 if the root was never expanded) */
  int32_t sum_n;
  int32_t noise_used;              /* Dirichlet draws consumed during the last search */
  int32_t sims_run;                /* simulations completed during the last search */
  uint16_t moves[CZ_MAX_MOVES];
  int32_t n[CZ_MAX_MOVES];         /* N(s,a) */
  double w[CZ_MAX_MOVES];          /* W(s,a) */
  float p[CZ_MAX_MOVES];           /* P(s,a) after legal-move renormalisation */
} cz_root_info;
/* node.a of the root (read by calc_policy, player.py:375-406).  Synchronises. */
int cz_get_root(cz_engine* e, int game, cz_root_info* out_host);

#define CZ_MAX_PV 32
typedef struct cz_pv_info {
  int32_t n_moves;
  int32_t has_value;               /* the position the line ends on has been evaluated (`state in self.debug`, player.py:436) */
  float value;                     /* its network value, from its side to move */
  uint16_t moves[CZ_MAX_PV];       /* canonical moves, each from its mover's point of view */
} cz_pv_info;
/* print_depth_info (player.py:408-450): most-visited line from the root of `game` (last maximum wins, the root skips its
 * no_act moves), at most max_len <= CZ_MAX_PV plies.  Synchronises. */
int cz_get_pv(cz_engine* e, int game, int32_t max_len, cz_pv_info* out_host);

/* Visit counts of every root after a search: n_host [n_games][CZ_MAX_MOVES], moves_host likewise
 * (0xFFFF padded), counts_host [n_games] legal-move counts, sims_run_host [n_games] or NULL.  Synchronises. */
int cz_get_root_stats(cz_engine* e, int32_t* n_host, uint16_t* moves_host, int32_t* counts_host, int32_t* sims_run_host);

/* Compact every game's pools now: keep the nodes reachable from the current root (statistics untouched), drop the
 * rest, rebuild the hash tables.  cz_search_begin does this on its own when a pool cannot hold the next search. */
int cz_compact(cz_engine* e);

/* Search statistics summed over all games since cz_create, for checking the byte model of the tree kernels (SURVEY.md
 * §8d): out[0] simulations backed up, out[1] sum of their path lengths (edges), out[2] simulations that ended without
 * the network (terminal, repetition, error), out[3] nodes created (= positions sent to the network), out[4] edges and
 * out[5] nodes currently stored (mean legal moves per node = out[4]/out[5]).  Synchronises. */
int cz_get_search_stats(cz_engine* e, uint64_t* out /* [6] */);

/* Counters since cz_create: [0] simulations completed, [1] NN positions evaluated, [2] wave iterations,
 * [3] finished-game records dropped because the ring was full (0 unless cz_play_move was driven without draining),
 * [4] whole-table resets (compaction was not enough / root unknown), [5] compactions,
 * [6] OR of the per-game error flags (1 path longer than max_path, 2 pool exhausted inside a search, 4 host noise table
 * exhausted, 8 node without a playable move), [7] number of games with a flag set.  Flags clear at cz_reset_games. */
int cz_get_counters(cz_engine* e, uint64_t* out_host /* [8] */);

/* ------------------------------------------------------------------------------------------
 * On-device self-play — worker/self_play.py:95-212 (start_game loop) for all games at once
 * ---------------------------------------------------------------------------------------- */
/* One ply for every live game: calc_policy + apply_temperature + sampling (player.py:375-406,
 * 453-470,195), new_step, draw / repetition / resign adjudication (self_play.py:126-175), final
 * move and value signs (:177-191).  Finished games are recorded and restarted from INIT_STATE.
 * n_finished counts games that ended in this call.  Synchronises. */
int cz_play_move(cz_engine* e, int32_t* n_finished);
/* Search + play until `target_games` games finished or `max_moves` plies were played.  Also returns early (with what it
 * did so far) when the finished-game ring could not take another ply's worth of records — drain it and call again — and
 * when every slot has retired (cz_config.game_quota). */
int cz_selfplay(cz_engine* e, int32_t target_games, int32_t max_moves, int32_t* games_done, int64_t* sims_done);

typedef struct cz_record_hdr {
  int32_t n_plies;      /* moves stored (including a final king capture) */
  int32_t value_red;    /* result from red's view: 1, -1, 0 (self_play.py:190-191) */
  int32_t game_index;   /* running index of the game on this engine */
  int32_t flags;        /* bit0 resign, bit1 draw by rule */
} cz_record_hdr;
/* Drain finished-game records into host memory: hdr_host [cap], moves_host [cap][max_plies+1]
 * (moves as seen by the side that played them, i.e. the strings self_play.py:132 appends).
 * Returns the number drained in *n.  Synchronises. */
int cz_drain_records(cz_engine* e, cz_record_hdr* hdr_host, uint16_t* moves_host, int32_t cap, int32_t* n);
/* Simulations per move of the games currently in the slots (per-game `simulation_num_per_move`, evaluator.py:153-154):
 * sims_host [n_games], 0 = cz_config.sims_per_move.  A slot keeps its value until its game ends.  Stream-ordered. */
int cz_set_game_sims(cz_engine* e, const int32_t* sims_host);
/* Which slots will search / play next: active_host [n_games] (arena: the slot of the player to move; 0 everywhere once
 * every slot has retired under cz_config.game_quota).  Synchronises. */
int cz_get_active(cz_engine* e, int32_t* active_host);
/* Device-side view of the same ring (for the NCCL gather of play records, SURVEY.md §8e). */
int cz_record_buffer(cz_engine* e, void** dev_ptr, uint64_t* bytes, int32_t* n_ready);
/* Layout of that ring for a peer that received it through the collective: out[0] = ring capacity in records, out[1] = uint16
 * slots per record row, out[2] = byte offset of the move rows inside the buffer (the headers start at 0, 16 bytes each),
 * out[3] = total bytes.  Host-only. */
int cz_record_layout(cz_engine* e, int64_t* out /* [4] */);
/* Forget the records in the ring (after a gather shipped them), and their visit pairs.  Stream-ordered. */
int cz_clear_records(cz_engine* e);
/* cz_config.record_visits engines: cz_drain_records plus every record's root visit counts, the policy calc_policy builds
 * (agent/player.py:375-406) that worker/self_play.py:112,134,178-180 keeps commented out.  ply_pairs_host [cap][max_plies+1]
 * u8: (label, N) pairs per ply, 0 for the appended final king capture (never searched; self_play.py:180 would one-hot it);
 * pairs_host [pair_cap][2] u32 (label, N): the records' plies in order, each ply's pairs in ascending label order, every
 * root edge with N > 0 (no_act moves are zeroed, player.py:381-383); labels index ActionLabelsRed in the mover's frame.
 * *n records, *n_pairs pairs.  Then clears the ring like cz_drain_records (which, on such an engine, drops the pairs).
 * Synchronises. */
int cz_drain_records_visits(cz_engine* e, cz_record_hdr* hdr_host, uint16_t* moves_host, uint8_t* ply_pairs_host,
                            uint32_t* pairs_host, int64_t pair_cap, int32_t cap, int32_t* n, int64_t* n_pairs);
/* Device-side view of the visit pairs beside the ring (record_visits engines; CZ_ERR_STATE otherwise): *dev_ptr the block,
 * *used_bytes its prefix that holds every pair of the records in the ring (what a gather ships).  Synchronises. */
int cz_record_visits_buffer(cz_engine* e, void** dev_ptr, uint64_t* used_bytes);
/* Layout of that block: bytes 0-7 u64 = pairs used; out[0] = byte offset of the first heap pair per ring slot (i64
 * [ring capacity]), out[1] = byte offset of the pairs per ply (u8 [ring capacity][uint16 slots per record row, see
 * cz_record_layout out[1]]), out[2] = byte offset of the pairs (u32 [][2] = label, N), out[3] = total bytes.  Host-only. */
int cz_record_visits_layout(cz_engine* e, int64_t* out /* [4] */);

/* ------------------------------------------------------------------------------------------
 * Policy + value network — agent/model.py:32-83 behind agent/api.py:37-74
 * ---------------------------------------------------------------------------------------- */
typedef struct cz_tensor_desc {
  const char* name;     /* Keras layer weight name, e.g. "res3_conv1-3-256/kernel" */
  const void* dev;      /* float32, Keras layout (conv HWIO, dense (in,out), vectors (C)) */
  int64_t numel;
} cz_tensor_desc;
/* Fold BatchNorm (eps 1e-3) into fp16 GEMM operands and upload; weights stay caller-owned. */
int cz_nn_set_weights(cz_engine* e, const cz_tensor_desc* descs, int32_t n);
/* Second network of the arena (net 0 = best model, net 1 = next generation; evaluator.py:31-40). */
int cz_nn_set_weights_net(cz_engine* e, int32_t net, const cz_tensor_desc* descs, int32_t n);
/* predict_on_batch (api.py:62-64): planes_dev [B][14][10][9] f32 ([B][28][10][9] with use_history) -> policy_dev
 * [B][2086] f32 (softmax), value_dev [B] f32 (tanh). */
int cz_nn_forward(cz_engine* e, const float* planes_dev, int32_t batch, float* policy_dev, float* value_dev);
/* Same from packed boards (plane encoding fused into the first convolution); with use_history every position is two
 * consecutive records: the board and the history board (all empty = zero planes). */
int cz_nn_forward_boards(cz_engine* e, const uint8_t* boards_dev, int32_t batch, float* policy_dev, float* value_dev);
/* Timing of the residual-tower tensor-core launches (the dominant kernel): while on, every network forward (cz_search's
 * included) brackets its tower with two one-thread kernels that read the device's %globaltimer.  Switches the bracketing
 * on/off and returns + clears what accumulated since the last call: device milliseconds, launches and algorithmic FLOPs
 * (2*90*9*C*C per position per launch, positions as counted on the device).  Synchronises. */
int cz_nn_profile(cz_engine* e, int enable, double* ms, uint64_t* launches, double* flops);
/* Kernel launches issued by this engine since creation (bench.py "gpu_launches"). */
int cz_launch_count(cz_engine* e, uint64_t* n);

/* ------------------------------------------------------------------------------------------
 * Tensor-core building blocks, exported for parity tests and profiling of the dominant kernel
 * (the residual-block convolutions of agent/model.py:68-83 and the policy Dense of :54).
 * ---------------------------------------------------------------------------------------- */
/* 3x3 "same" convolution + bias (+ residual) (+ ReLU) on fp16 activations [n_boards][10][9][c], fed by im2col-mode TMA;
 * w fp16 [9][c][c] = [tap kh*3+kw][c_out][c_in]; bias f32 [c]. */
int cz_igemm_conv3x3_dense(const void* act_in_dev, const void* w_dev, const float* bias_dev, const void* residual_dev,
                           void* act_out_dev, int n_boards, int c, int relu, void* stream);
/* `count` draws of the on-device root-noise sampler (noise_mode 1): the first component of
 * Dirichlet(alpha * 1_n_moves), i.e. what np.random.dirichlet(alpha*ones(n))[0] (player.py:304) is distributed as: draws
 * 0 .. count-1 of the stream slot `game` is on (it moves to a new stream with every search opened on the slot). */
int cz_noise_sample(cz_engine* e, int game, int n_moves, int count, double* out_dev);
/* out[m][n] = sum_k a[m][k] * w[n][k] + bias[n]; a fp16 [m][k], w fp16 [n_pad][k], bias f32 [n_pad] (padded like w),
 * out f32 [m][ldo], 16-byte aligned with ldo a multiple of 4. */
int cz_igemm_dense(const void* a_dev, const void* w_dev, const float* bias_dev, float* out_dev, int m, int n_valid,
                   int n_pad, int k, int n_tile, int ldo, void* stream);
/* Intermediate buffers of the network forward, as the last cz_nn_forward / cz_nn_forward_boards left them (dense layout;
 * rows = positions, C = nn_filters):
 *   FIRST_OUT    fp16 [90][C]  first convolution + BN + ReLU (1-block nets only: deeper towers overwrite it)
 *   FIRST_OUT32  f32  [90][C]  its fp32 skip-stream copy (fp32 skip stream and 1 block only)
 *   LAST_CONV1   fp16 [90][C]  first convolution of the last residual block
 *   TOWER_OUT    fp16 [90][C]  output of the residual tower (what the heads read)
 *   TOWER_OUT32  f32  [90][C]  its fp32 skip-stream copy (fp32 skip stream only; the heads read this one then)
 *   POL_FEAT     fp16 [3 * pol_k1]  policy features split as [hi | lo | hi], pol_k1 = policy channels * 90 padded to 64
 *   LOGITS       f32  [2304]   policy logits (labels 2086.. are padding)
 *   STATS        float2 [9]    per 256-label tile {max logit, sum exp(logit - max)} of the policy GEMM epilogue */
typedef enum cz_nn_buffer {
  CZ_NN_BUF_FIRST_OUT = 0,
  CZ_NN_BUF_FIRST_OUT32 = 1,
  CZ_NN_BUF_LAST_CONV1 = 2,
  CZ_NN_BUF_TOWER_OUT = 3,
  CZ_NN_BUF_TOWER_OUT32 = 4,
  CZ_NN_BUF_POL_FEAT = 5,
  CZ_NN_BUF_LOGITS = 6,
  CZ_NN_BUF_STATS = 7
} cz_nn_buffer;
/* Copy the first n position rows of buffer `which` (cz_nn_buffer) to dst_dev; *row_bytes = bytes per row.  dst_dev = NULL
 * only reports row_bytes.  CZ_ERR_ARG: unknown buffer, n > max batch or dst_bytes < n * row_bytes; CZ_ERR_STATE: the
 * buffer does not exist in this configuration.  Synchronises. */
int cz_nn_read_buffer(cz_engine* e, int32_t which, int32_t n, void* dst_dev, int64_t dst_bytes, int64_t* row_bytes);

/* ------------------------------------------------------------------------------------------
 * Training — one Keras Model.fit batch of worker/optimize.py:108-136 (SGD momentum, categorical cross-entropy + MSE
 * + L2, BatchNormalization in training mode).  Same conventions as the engine: one caller-owned device workspace
 * (cz_train_workspace_bytes), caller-owned device tensors passed by pointer, stream-ordered calls, a negative cz_status
 * with a message in cz_last_error() on error.
 * ---------------------------------------------------------------------------------------- */
typedef struct cz_trainer cz_trainer;
typedef struct cz_train_config {
  int32_t struct_bytes;        /* sizeof(cz_train_config) */
  int32_t filters;             /* cnn_filter_num: 64..256, multiple of 64 */
  int32_t blocks;              /* res_layer_num */
  int32_t in_planes;           /* 14, or 28 with use_history */
  int32_t policy_channels;     /* 1x1 policy conv filters (agent/model.py: 4; legacy configs 2 or 32) */
  int32_t value_channels;      /* 1x1 value conv filters (2; legacy 4) */
  int32_t value_fc;            /* value_fc_size, <= 256 */
  int32_t max_batch;           /* largest batch of cz_train_step, <= 4096 */
} cz_train_config;
typedef struct cz_train_hparams {
  int32_t struct_bytes;        /* sizeof(cz_train_hparams) */
  float lr, momentum;          /* SGD: v = momentum * v - lr * g; w += v */
  float w_policy, w_value;     /* config.trainer.loss_weights */
  float l2;                    /* config.model.l2_reg: loss += l2 * sum K^2 over conv and Dense kernels */
} cz_train_hparams;
int cz_train_workspace_bytes(const cz_train_config* cfg, uint64_t* bytes);
int cz_train_create(const cz_train_config* cfg, void* workspace_dev, uint64_t bytes, void* stream, cz_trainer** out);
void cz_train_destroy(cz_trainer* t);
/* params: every weight in Keras names and layouts (f32, including BN moving_mean / moving_variance); velocity: one
 * tensor per trainable weight (kernels, biases, BN gamma / beta), same names and sizes.  cz_train_step updates both IN
 * PLACE (and the moving statistics).  CZ_ERR_ARG: a tensor is missing or has the wrong size. */
int cz_train_set_params(cz_trainer* t, const cz_tensor_desc* params, int32_t n, const cz_tensor_desc* velocity, int32_t n_velocity);
/* One step on `batch` samples: planes_dev [B][in_planes][10][9] f32 (one-hot), policy_target_dev [B][2086] f32,
 * value_target_dev [B] f32.  losses_dev[4] f32 = {total, policy cross-entropy, value MSE, l2 term} before the update.
 * CZ_ERR_ARG: batch outside 1..max_batch; CZ_ERR_STATE: no parameters set.  Bit-reproducible. */
int cz_train_step(cz_trainer* t, const float* planes_dev, const float* policy_target_dev, const float* value_target_dev,
                  int32_t batch, const cz_train_hparams* hp, float* losses_dev);
/* Tests: copy the last step's gradient of one trainable weight (loss terms only, without the L2 part).  CZ_ERR_ARG:
 * unknown name or numel differs.  Synchronises; off the step path. */
int cz_train_read_grad(cz_trainer* t, const char* name, void* dst_dev, int64_t numel);
/* Tests: intermediate buffers of the training step, as the LAST cz_train_step left them (n = that step's batch, P = n * 90,
 * C = filters, L = blocks, pc / vc = policy / value channels, H = value_fc).  `index` selects a block or a BN layer
 * (0 = input, 1 + 2i + j = block i conv j + 1, 2L + 1 = policy, 2L + 2 = value) and is 0 for every other buffer.
 *   PLANE_INDEX     int8 [n][2][90]  occupied plane 0..13 per (position, board, pixel), -1 empty (board 1: 28 planes only)
 *   BLOCK_OUT32     f32  [P][C]      k = 0..L: output of the input conv (k = 0) / of block k, the skip stream
 *   BLOCK_OUT16     fp16 [P][C]      k = 0..L: the same activations in fp16 (conv and wgrad operands)
 *   CONV1_OUT16     fp16 [P][C]      i < L: relu(BN(conv1)) of block i
 *   BN_MEAN         f32  [C_j]       batch mean of BN layer j
 *   BN_VAR          f32  [C_j]       biased batch variance of BN layer j
 *   BN_DZ           f32  [P][C_j]    the gradient at BN layer j's input: the backward writes dz over the conv output z
 *   POL_FEAT        f32  [n][pc*90]  relu(BN(policy conv)) in Keras Flatten order (channel * 90 + pixel)
 *   VAL_FEAT        f32  [n][vc*90]  the value features, same order
 *   LOGITS, DLOGITS f32  [n][2086]   policy logits / the loss gradient at the logits (w_policy / n included)
 *   VAL_HIDDEN_PRE  f32  [n][H]      value_dense before the ReLU
 *   VAL_HIDDEN      f32  [n][H]      after the ReLU
 *   DVAL_HIDDEN     f32  [n][H]      gradient at VAL_HIDDEN, masked by VAL_HIDDEN_PRE > 0 (the gradient at value_dense)
 *   VAL_PRE         f32  [n]         value before tanh;  DVAL_PRE  f32 [n]  the loss gradient at it
 *   CE_ROWS         f32  [n]         per-row cross-entropy;  SE_ROWS  f32 [n]  per-row squared value error
 *   DPOL_FEAT       f32  [n][pc*90]  gradient at POL_FEAT (Flatten order); the value's feature gradient was overwritten
 *   TRUNK_GRAD      f32  [P][C]      gradient at BLOCK_OUT32[0] (before the input BN's ReLU mask)
 *   SCALE_SLOTS     f32  [2L+1][4]   per 3x3 conv 2i + j: {max |dz| as float bits, 2^e, 2^-e, unused} of its fp16 dz
 * dst_dev = NULL only reports *bytes.  CZ_ERR_ARG: unknown buffer, index out of range or dst_bytes < *bytes;
 * CZ_ERR_STATE: no step has run.  Synchronises; off the step path. */
typedef enum cz_train_buffer {
  CZ_TRAIN_BUF_PLANE_INDEX = 0,
  CZ_TRAIN_BUF_BLOCK_OUT32 = 1,
  CZ_TRAIN_BUF_BLOCK_OUT16 = 2,
  CZ_TRAIN_BUF_CONV1_OUT16 = 3,
  CZ_TRAIN_BUF_BN_MEAN = 4,
  CZ_TRAIN_BUF_BN_VAR = 5,
  CZ_TRAIN_BUF_BN_DZ = 6,
  CZ_TRAIN_BUF_POL_FEAT = 7,
  CZ_TRAIN_BUF_VAL_FEAT = 8,
  CZ_TRAIN_BUF_LOGITS = 9,
  CZ_TRAIN_BUF_DLOGITS = 10,
  CZ_TRAIN_BUF_VAL_HIDDEN_PRE = 11,
  CZ_TRAIN_BUF_VAL_HIDDEN = 12,
  CZ_TRAIN_BUF_DVAL_HIDDEN = 13,
  CZ_TRAIN_BUF_VAL_PRE = 14,
  CZ_TRAIN_BUF_DVAL_PRE = 15,
  CZ_TRAIN_BUF_CE_ROWS = 16,
  CZ_TRAIN_BUF_SE_ROWS = 17,
  CZ_TRAIN_BUF_DPOL_FEAT = 18,
  CZ_TRAIN_BUF_TRUNK_GRAD = 19,
  CZ_TRAIN_BUF_SCALE_SLOTS = 20
} cz_train_buffer;
int cz_train_read_buffer(cz_trainer* t, int32_t which, int32_t index, void* dst_dev, int64_t dst_bytes, int64_t* bytes);
/* Switches the trainer to Keras 2.0.8 Adam (decay 0; worker/sl.py, worker/sl_onegreen.py).  m / v: one f32 tensor per
 * trainable weight, named and sized like the velocity of cz_train_set_params; cz_train_step updates them IN PLACE, reads
 * hp->lr as Keras' base lr and ignores hp->momentum.  Every trainable tensor is updated by ONE fused launch:
 *   t = iterations + 1;  lr_t = fp32(lr * (sqrt(1 - beta_2^t) / (1 - beta_1^t)))  (float64)
 *   g = grad + 2 l2 K (kernels only);  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g g;  w -= (lr_t m) / (sqrt(v) + eps)
 * in fp32 without contraction, b1 = fp32(beta_1), 1 - b1 in fp32.  Resets iterations to 0; every successful
 * cz_train_step adds 1.  A later cz_train_set_params returns the trainer to SGD.  CZ_ERR_STATE: no parameters set;
 * CZ_ERR_ARG: a moment is missing or mis-sized, or beta / epsilon out of range. */
int cz_train_set_adam(cz_trainer* t, const cz_tensor_desc* m, int32_t n_m, const cz_tensor_desc* v, int32_t n_v, double beta_1,
                      double beta_2, double epsilon);
/* Adam's step counter (Keras `iterations`).  CZ_ERR_STATE: the trainer uses SGD. */
int cz_train_adam_iterations(cz_trainer* t, int64_t* iterations);
/* Stage building blocks of the step, for parity tests (allocate scratch, synchronise):
 *   wgrad3x3  dw (Keras HWIO [3][3][c][c] f32) of a 3x3 "same" conv: x16 fp16 [n][10][9][c], dy f32 [n*90][c]
 *   dgrad3x3  dx f32 [n*90][c] = input gradient of that conv for HWIO weights w_hwio f32
 *   bn        training-mode BN (+ skip) + ReLU on z [rows][c]: out, batch mean, biased var; with up (gradient of the
 *             ReLU output) also dz, dgamma, dbeta */
int cz_train_wgrad3x3(const void* x16_dev, const float* dy_dev, int n, int c, float* dw_dev, void* stream);
int cz_train_dgrad3x3(const float* dy_dev, const float* w_hwio_dev, int n, int c, float* dx_dev, void* stream);
int cz_train_bn(const float* z_dev, long long rows, int c, const float* gamma_dev, const float* beta_dev, const float* skip_dev,
                float* out_dev, float* mean_dev, float* var_dev, const float* up_dev, float* dz_dev, float* dgamma_dev,
                float* dbeta_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CCZERO_B200_H */
