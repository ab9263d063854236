"""What the REAL reference computes for the inputs of tests/test_oracle_vs_reference.py -> tests/golden/reference_pins.json.gz.
Needs the reference tree (oracle/ref_import.py); the tests then compare the oracle restatements with these vectors anywhere.

    python -m oracle.gen_golden_pins
"""
import gzip
import hashlib
import json
import os
import random

import numpy as np

from . import ref_import
from . import senv as o

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
OUT = os.path.join(GOLD, "reference_pins.json.gz")


def planes_digest(p):
    return hashlib.sha256(np.ascontiguousarray(np.asarray(p, dtype=np.float32)).tobytes()).hexdigest()[:16]


def array_digest(a):
    a = np.ascontiguousarray(a)
    return [list(a.shape), str(a.dtype), hashlib.sha256(a.tobytes()).hexdigest()]


def position_row(r, s, m=None, catch=True):
    """Everything the env tests compare at state `s` (and move `m`), computed by the reference's static_env."""
    row = {"s": s, "lm": r.get_legal_moves(s), "done": list(r.done(s)), "done_check": list(r.done(s, need_check=True)),
           "planes": planes_digest(r.state_to_planes(s)), "attack": r.has_attack_chessman(s), "flip": r.fliped_state(s)}
    if m is not None:
        row["m"] = m
        row["new_step"] = r.new_step(s, m)
        if catch:
            row["wcc"] = r.will_check_or_catch(s, m)
            row["catched"] = r.be_catched(s, m)
    return row


def random_playouts(r):
    rng = random.Random(7)
    games = []
    for g in range(25):
        s, rows = r.INIT_STATE, []
        for ply in range(200):
            lm = r.get_legal_moves(s)
            if r.done(s)[0]:
                rows.append(position_row(r, s))
                break
            m = rng.choice(lm)
            rows.append(position_row(r, s, m, catch=ply % 2 == 0))
            s = r.step(s, m)
        games.append(rows)
    return games


def arbitrary_boards(r):
    from tests.env_checks import EXTREME_STATES, random_boards
    rows = []
    for s in random_boards(600, 5) + [x for x in EXTREME_STATES if 's' in x and 'S' in x]:
        lm = r.get_legal_moves(s)
        m = lm[len(s) % len(lm)] if lm and not r.done(s)[0] else None
        rows.append(position_row(r, s, m))
    return rows


def main():
    r = ref_import.senv()
    lt = ref_import.lookup_tables()
    out = {"generator": "oracle/gen_golden_pins.py",
           "labels": lt.ActionLabelsRed, "flip50": [lt.flip_move(m) for m in lt.ActionLabelsRed[:50]],
           "playouts": random_playouts(r), "boards": arbitrary_boards(r)}
    s = '4s4/9/4e4/p8/2e2R2p/P5E2/8P/9/9/4S1E2'
    out["fen"] = [[st, t, r.state_to_fen(st, t), r.fen_to_state(r.state_to_fen(st, t))]
                  for st, t in ((o.INIT_STATE, 0), (o.step(o.INIT_STATE, '0001'), 1), (s, 7), (s, 10))]

    from .ref_player_harness import real_player_moves
    out["player_k1"] = []
    for sims, seed in ((80, 1), (150, 2)):
        a, edges, sum_n = real_player_moves([(o.INIT_STATE, 0, None, False)], sims, seed)[0]
        out["player_k1"].append({"sims": sims, "seed": seed, "action": a, "sum_n": sum_n,
                                 "edges": {m: [int(e[0]), float(e[1]), float(e[2]), float(e[3])] for m, e in edges.items()}})
    lm = o.get_legal_moves(o.INIT_STATE)
    out["player_k10"] = {"sims": 300, "search_threads": 10, "moves": lm, "visits": [
        [int(x[1].get(m, (0,))[0]) for m in lm] for x in
        (real_player_moves([(o.INIT_STATE, 0, None, False)], 300, seed, search_threads=10)[0] for seed in range(5))]}

    from . import ref_worker_harness as h
    play = dict(max_game_length=20, tau_decay_rate=0.98, noise_eps=0.25, enable_resign_rate=0.1, resign_threshold=-0.5, min_resign_turn=4)
    out["game_loops"] = {"play": play,
                         "selfplay": [{"seed": seed, **h.real_selfplay_game(seed, 16, **play)} for seed in (41, 42)],
                         "arena": [{"seed": seed, "idx": idx, **h.real_arena_game(seed, idx, 16, **play)} for seed, idx in ((43, 0), (44, 1))]}

    _, ev = h.worker_modules()
    cfg = ref_import.config("mini")
    results = [1, -1, 0, 1, 1, -1, 0, 0, -1, 1, 1, -1]
    cfg.eval.game_num = len(results)
    w = ev.EvaluateWorker(cfg, pid=0)
    w.start_game = lambda idx: (results[idx], 40)
    sleep, ev.sleep = ev.sleep, (lambda s: None)
    try:
        out["tally"] = {"results": results, "want": list(w.start())}
    finally:
        ev.sleep = sleep

    import cchess_alphazero.worker.optimize as ropt
    from cczero_b200.records import record_to_play_data
    with gzip.open(os.path.join(GOLD, "games_k1.json.gz"), "rt") as f:
        game = next(g for g in json.load(f)["games"] if g["kind"] == "selfplay" and g["result"]["moves"] and g["result"]["value_red"] != 0)
    data = record_to_play_data({"moves": game["result"]["moves"], "value_red": game["result"]["value_red"]})
    out["expanding_data"] = {str(int(hist)): [array_digest(x) for x in ropt.expanding_data(data, hist)] for hist in (False, True)}

    from . import keras_graph, model as om
    from tests.search_checks import game_history
    w28 = om.init_weights(128, 7, 256, seed=2, trained_like=True, spread=0.5, in_planes=28, policy_filters=32, value_filters=4)
    hists = [game_history(n, 30 + n) for n in (2, 5, 17, 40)]
    p28 = np.stack([o.state_history_to_planes(hh[-1], hh) for hh in hists])
    gp, gv = keras_graph.run(os.path.join(ref_import.REF_ROOT, "data", "model", "model_128_l1_config.json"), w28, p28)
    out["keras_graph_28"] = {"policy": np.asarray(gp, np.float64).tolist(), "value": np.asarray(gv, np.float64)[:, 0].tolist()}

    with gzip.open(OUT, "wt") as f:
        json.dump(out, f)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
