"""`worker.evaluator` drop-in (reference: cchess_alphazero/worker/evaluator.py:28-250): best model vs next generation.

`start(config)` keeps the reference's role: load both models, play `config.eval.game_num * config.play.max_processes`
games with alternating colours, report the next generation's score.  Where the reference runs processes with two
`CChessPlayer`s each, all games run concurrently in ONE arena engine (`cz_config.arena`): per game two search trees (one
per player), network 0 = best model, network 1 = next generation, evaluator draw rules, all on the GPU.
`config.play` must already carry the evaluation settings (`config.eval.update_play_config(config.play)`, manager.py:102).
"""
from logging import getLogger

from .engine import Engine
from .model import engine_net_kwargs
from .lib import get_lib

logger = getLogger(__name__)


def score_for_next_generation(value_red, idx):
    """evaluator.py:127-137: the best model is red in even games."""
    score = 0 if value_red == -1 else (1 if value_red == 1 else 0.5)
    return 1 - score if idx % 2 == 0 else score


def tally_games(results):
    """EvaluateWorker.start's bookkeeping (evaluator.py:93-145) over (game index, red's result) pairs:
    (total_score, red_new_win, red_new_draw, red_new_fail, black_new_win, black_new_draw, black_new_fail)."""
    tally = {"red": [0, 0, 0], "black": [0, 0, 0]}           # next generation as red / black: win, draw, fail
    total = 0
    for idx, v in results:
        ng_is_red = idx % 2 == 1
        ng_result = v if ng_is_red else -v                   # +1 win, 0 draw, -1 fail for the next generation
        tally["red" if ng_is_red else "black"][{1: 0, 0: 1, -1: 2}[ng_result]] += 1
        total += score_for_next_generation(v, idx)
    r, b = tally["red"], tally["black"]
    return (total, r[0], r[1], r[2], b[0], b[1], b[2])


class EvaluateWorker:
    def __init__(self, config, model_bt, model_ng, n_games=None, concurrent_games=None, lib=None, device=None, seed=0,
                 playouts=(8, 12), eval_mirror=False):
        """playouts: every game draws `randint(lo, hi) * 100` simulations per move when it starts (evaluator.py:153-154);
        None = config.play.simulation_num_per_move for every game.  eval_mirror: each side's network averages every leaf
        and its left-right mirror."""
        self.config = config
        pc, mc = config.play, config.model
        self.n_games = n_games or config.eval.game_num * pc.max_processes
        m = concurrent_games or min(self.n_games, 512)
        self.m = m
        sims_max = playouts[1] * 100 if playouts else pc.simulation_num_per_move
        self.engine = Engine(
            lib or get_lib(), device, n_games=2 * m, sims_per_move=pc.simulation_num_per_move,
            leaves_per_round=pc.search_threads, virtual_loss=getattr(pc, "virtual_loss", 3), noise_mode=1, c_puct=pc.c_puct,
            noise_eps=pc.noise_eps, dirichlet_alpha=getattr(pc, "dirichlet_alpha", 0.2), tau_decay_rate=pc.tau_decay_rate,
            enable_resign_rate=0.0, max_game_length=pc.max_game_length, max_nodes_per_game=max(4096, 16 * sims_max),
            seed=seed, arena=True, **engine_net_kwargs(mc),
            game_quota=self.n_games, playouts=playouts, eval_mirror=eval_mirror)   # exactly the games 0 .. n_games-1, each played to its end
        self.engine.set_weights(model_bt.torch_weights(), net=0)
        self.engine.set_weights(model_ng.torch_weights(), net=1)
        self.engine.reset()

    def start(self):
        """Returns (total_score, red_new_win, red_new_draw, red_new_fail, black_new_win, black_new_draw, black_new_fail)
        like EvaluateWorker.start (evaluator.py:93-145): the games with running index 0 .. n_games-1 (`for idx in
        range(game_num)`, :104), every one played to its end — a slot whose next game would be past the quota retires
        (cz_config.game_quota) instead of starting games nobody counts, so quick decisive games are not over-sampled."""
        results = {}
        while len(results) < self.n_games:
            done, sims = self.engine.selfplay(target_games=self.n_games - len(results), max_moves=0)
            recs = self.engine.drain_records()
            for rec in recs:
                assert rec["game_index"] < self.n_games and rec["game_index"] not in results
                results[rec["game_index"]] = rec["value_red"]
            if not recs and sims == 0:
                raise RuntimeError(f"arena stalled: {len(results)} of {self.n_games} games finished and no slot is active")
        return tally_games(sorted(results.items()))

    def close(self):
        self.engine.close()


def start(config, model_bt=None, model_ng=None, eval_mirror=False):
    """evaluator.py:28-82."""
    from .model import CChessModel
    rc = config.resource
    if model_bt is None:
        model_bt = CChessModel(config)
        if not model_bt.load(rc.model_best_config_path, rc.model_best_weight_path):
            raise FileNotFoundError("best model not found")
    if model_ng is None:
        model_ng = CChessModel(config)
        if not model_ng.load(rc.next_generation_config_path, rc.next_generation_weight_path):
            raise FileNotFoundError("next generation model not found")
    worker = EvaluateWorker(config, model_bt, model_ng, eval_mirror=eval_mirror)
    total_score, rw, rd, rf, bw, bd, bf = worker.start()
    game_num = worker.n_games
    worker.close()
    win_rate = total_score * 100 / game_num
    logger.info(f"Evaluate over, next generation win {total_score}/{game_num} = {win_rate:.2f}%")
    logger.info(f"new red: {rw}/{rd}/{rf}  new black: {bw}/{bd}/{bf} (win/draw/fail)")
    return total_score, game_num
