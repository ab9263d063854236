"""Cost of the left-right mirror on one GPU.

Search: simulations/s of one whole `cz_search` at BASELINE config 3 (1024 games, 800 sims, K = 8, 20x256) and config 2
(256 games, 200 sims, 7x128) with `eval_mirror` off and on, alternated, and the residual tower's achieved TFLOP/s in the
mirrored form (cz_nn_profile over one more search; the positions counted are the leaves and their mirrors).

Training: one device batch's assembly (SlDataset.batch: gather, cz_env_mirror,
cz_env_encode_planes, policy target) without and with per-sample mirror flags, alternated, at 14 and 28 planes, against
one cz_train_step of a 10x192 network at the same batch size.  Prints one JSON line with the card's name, power limit
and SM clock, read in the same run.

    python tools/bench_mirror.py [--batch 512] [--reps 50] [--rounds 3]

The samples are seeded engine self-play games (random 64x2 net, 8 simulations per move), replayed into a device
dataset.  Nothing is written.
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cczero_b200  # noqa: E402,F401
from cczero_b200 import records as rd  # noqa: E402
from cczero_b200.env import StaticEnv  # noqa: E402
from cczero_b200.lib import get_lib  # noqa: E402
from oracle import model as om  # noqa: E402
from tools.bench_optimize_data import event_ms, selfplay_records  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power.limit": "not readable"}


SEARCH = {"c3": (1024, 800, 8, 256, 20), "c2": (256, 200, 8, 128, 7)}


def search_rates(lib, games, sims, k, filters, blocks, runs):
    import time
    from cczero_b200.engine import Engine
    w = {kk: torch.as_tensor(v) for kk, v in om.init_weights(filters, blocks, 256, seed=1).items()}
    engines = {}
    for mirror in (False, True):
        e = Engine(lib, "cuda", n_games=games, sims_per_move=sims, leaves_per_round=k, nn_filters=filters, nn_blocks=blocks,
                   seed=3, max_nodes_per_game=max(4096, 24 * sims), eval_mirror=mirror)
        e.set_weights(w)
        e.reset()
        e.search(None)                                       # first search: module load and the graph capture
        engines[mirror] = e
    rates = {False: [], True: []}
    for _ in range(runs):
        for mirror in (False, True):
            e = engines[mirror]
            e.reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e.search(None)
            torch.cuda.synchronize()
            rates[mirror].append(float(e.sims_run().sum()) / (time.perf_counter() - t0))
    e = engines[True]
    e.nn_profile(True)
    e.reset()
    e.search(None)
    ms, launches, flops = e.nn_profile(False)
    for e in engines.values():
        e.close()
    return {"sims_per_s_off": rates[False], "sims_per_s_on": rates[True],
            "on_over_off": float(np.median(rates[True]) / np.median(rates[False])),
            "tower_tflops_mirrored": flops / (ms * 1e-3) / 1e12, "tower_launches": launches}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=50, help="batches per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="alternated plain / mirrored windows")
    ap.add_argument("--games", type=int, default=200)
    ap.add_argument("--search-runs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from cczero_b200.model import CChessModel
    from cczero_b200.train import Trainer
    lib = get_lib()
    env = StaticEnv(lib, "cuda")
    games = [g for d in selfplay_records(lib, args.games, seed=1) for g in rd.split_games(d) if len(g) > 1]
    ds = rd.replay_play_games(lib, env.device, rd.pack_play_games(games, "bench"), env.label_lut)
    rng = np.random.RandomState(0)
    idx = rng.permutation(len(ds))[:args.batch]
    flags = rng.randint(0, 2, len(idx))
    out = {"card": card(), "positions": len(ds), "batch": len(idx)}
    out["search"] = {name: search_rates(lib, *shape, runs=args.search_runs) for name, shape in SEARCH.items()}
    for history in (False, True):
        n = 28 if history else 14
        plain, mirrored = [], []
        for _ in range(args.rounds):
            plain.append(event_ms(lambda: ds.batch(env, idx, history), args.reps))
            mirrored.append(event_ms(lambda: ds.batch(env, idx, history, mirror=flags), args.reps))
        mc = SimpleNamespace(cnn_filter_num=192, res_layer_num=10, value_fc_size=256, l2_reg=1e-4, input_depth=n,
                             policy_channels=4, value_channels=2, cnn_first_filter_size=5, cnn_filter_size=3)
        m = CChessModel(SimpleNamespace(model=mc, trainer=SimpleNamespace(momentum=0.9, loss_weights=[1.0, 1.0])))
        m.weights = om.init_weights(192, 10, 256, seed=1, in_planes=n)
        tr = Trainer(m, len(idx), "cuda")
        planes, pol, val = ds.batch(env, idx, history, mirror=flags)
        step = event_ms(lambda: tr.step_async(planes, pol, val, 1e-3), args.reps)
        tr.close()
        out[f"planes_{n}"] = {"batch_ms": plain, "batch_mirror_ms": mirrored, "train_step_ms_10x192": step,
                              "mirror_extra_share_of_step": (min(mirrored) - min(plain)) / step}
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
