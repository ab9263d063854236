"""Cost of recording root visit counts (cz_config.record_visits) and of training on them, on one GPU:

  * c3 self-play (1024 games, 800 simulations per move, 256x20 random net, K = 8) in simulations per second with
    recording on and off, alternated runs, the card's name, power limit and SM clock read in the same process;
  * the workspace bytes recording adds at that shape;
  * JSON bytes per game of the play-data files with and without visits (seeded 64x2 self-play games, 8 simulations);
  * `fill_queue` time for the same files on the device path with policy_target "move" and "visits", alternated;
  * device bytes per position of both datasets;
  * one batch's visit targets (cz_visit_targets) against one cz_train_step at 10x192 @ 512.

    python tools/bench_visit_records.py [--runs 3] [--plies 3] [--warmup 1] [--files 100]

Everything it writes goes to a temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from collections import deque
from random import Random
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cczero_b200  # noqa: E402,F401
from cczero_b200 import records as rd  # noqa: E402
from cczero_b200.engine import Engine  # noqa: E402
from cczero_b200.env import StaticEnv  # noqa: E402
from cczero_b200.lib import get_lib  # noqa: E402
from oracle import model as om  # noqa: E402
from tools.bench_optimize_data import event_ms  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit and clocks not readable"


def c3_rate(lib, weights, record_visits, plies, warmup):
    """Simulations per second of `plies` self-play plies after `warmup` plies, records drained every ply."""
    eng = Engine(lib, "cuda", n_games=1024, sims_per_move=800, leaves_per_round=8, nn_filters=256, nn_blocks=20,
                 max_nodes_per_game=24 * 800, seed=0, record_visits=record_visits)
    eng.set_weights(weights)
    eng.reset()
    for _ in range(warmup):
        eng.selfplay(target_games=0, max_moves=1)
        eng.drain_records()
    torch.cuda.synchronize()
    t0, sims = time.perf_counter(), 0
    for _ in range(plies):
        sims += eng.selfplay(target_games=0, max_moves=1)[1]
        eng.drain_records()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    ws = eng.workspace_bytes
    eng.close()
    return sims / dt, ws


def selfplay_records(lib, n_games, seed):
    w = om.init_weights(64, 2, 256, seed=seed)
    eng = Engine(lib, "cuda", n_games=n_games, sims_per_move=8, leaves_per_round=4, nn_filters=64, nn_blocks=2,
                 max_game_length=100, seed=seed, enable_resign_rate=0.0, record_visits=True)
    eng.set_weights({k: torch.as_tensor(v) for k, v in w.items()})
    eng.reset()
    recs = []
    while len(recs) < n_games:
        eng.selfplay(target_games=n_games - len(recs), max_moves=0)
        recs += eng.drain_records()
    eng.close()
    return [rd.record_to_play_data(r) for r in sorted(recs, key=lambda r: r["game_index"])[:n_games]]


def time_fill(env, files, target, seed):
    from cczero_b200.optimize import OptimizeWorker
    cfg = SimpleNamespace(trainer=SimpleNamespace(dataset_size=10 ** 9, batch_size=512),
                          opts=SimpleNamespace(has_history=False))
    w = OptimizeWorker(cfg, env=env, device="cuda", dataset="device", policy_target=target)
    w.filenames = deque(files)
    Random(seed).shuffle(w.filenames)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    w.fill_queue()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, w.dataset


def dataset_bytes(ds):
    cols = [ds.boards, ds.labels, ds.values, ds.ply] + (list(ds.visits) if ds.visits is not None else [])
    return sum(x.numel() * x.element_size() for x in cols) / len(ds)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3, help="alternated c3 runs per setting")
    ap.add_argument("--plies", type=int, default=3, help="timed plies per c3 run")
    ap.add_argument("--warmup", type=int, default=1, help="untimed plies per c3 run")
    ap.add_argument("--files", type=int, default=100, help="play-data files of 5 games for fill_queue")
    ap.add_argument("--reps", type=int, default=3, help="alternated fill_queue runs per target")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    lib = get_lib()
    res = {"card_before": card()}
    print(json.dumps(res), flush=True)

    w = {k: torch.as_tensor(v) for k, v in om.init_weights(256, 20, 256, seed=0).items()}
    rates = {"on": [], "off": []}
    for r in range(args.runs):
        for mode in (("off", "on") if r % 2 == 0 else ("on", "off")):
            rate, ws = c3_rate(lib, w, mode == "on", args.plies, args.warmup)
            rates[mode].append(rate)
            res[f"workspace_bytes_{mode}"] = ws
            print(json.dumps({"c3_run": r, "record_visits": mode, "sims_per_s": rate}), flush=True)
    res["c3_sims_per_s"] = rates
    res["c3_recording_overhead"] = 1 - np.median(rates["on"]) / np.median(rates["off"])
    res["workspace_bytes_added"] = res["workspace_bytes_on"] - res["workspace_bytes_off"]
    res["card_after_c3"] = card()
    print(json.dumps({k: res[k] for k in ("c3_sims_per_s", "c3_recording_overhead", "workspace_bytes_added", "card_after_c3")}),
          flush=True)

    env = StaticEnv(lib, "cuda")
    recs = selfplay_records(lib, args.files * 5, seed=1)
    plain = [[it if isinstance(it, str) else it[:2] for it in g] for g in recs]
    res["json_bytes_per_game"] = {"with_visits": len(json.dumps(recs)) / len(recs), "without": len(json.dumps(plain)) / len(plain)}
    res["positions"] = sum(len(g) - 1 for g in recs)
    with tempfile.TemporaryDirectory() as d:
        files = []
        for i in range(args.files):
            p = os.path.join(d, f"play_{i:05d}.json")
            with open(p, "w") as f:
                json.dump(sum(recs[5 * i:5 * i + 5], []), f)
            files.append(p)
        times = {"move": [], "visits": []}
        time_fill(env, files[:2], "move", 0)
        time_fill(env, files[:2], "visits", 0)
        for r in range(args.reps):
            for target in (("move", "visits") if r % 2 == 0 else ("visits", "move")):
                t, ds = time_fill(env, files, target, r)
                times[target].append(t)
                res[f"device_bytes_per_position_{target}"] = dataset_bytes(ds)
                if target == "visits":
                    vds = ds
        res["fill_queue_s"] = times
    print(json.dumps({k: res[k] for k in ("json_bytes_per_game", "positions", "fill_queue_s", "device_bytes_per_position_move",
                                          "device_bytes_per_position_visits")}), flush=True)

    from cczero_b200.model import CChessModel
    from cczero_b200.train import Trainer
    bs = 512
    idx = np.random.RandomState(0).permutation(len(vds))[:bs]
    ids = torch.as_tensor(idx, device="cuda")
    mc = SimpleNamespace(cnn_filter_num=192, res_layer_num=10, value_fc_size=256, l2_reg=1e-4, input_depth=14, policy_channels=4,
                         value_channels=2, cnn_first_filter_size=5, cnn_filter_size=3)
    m = CChessModel(SimpleNamespace(model=mc, trainer=SimpleNamespace(momentum=0.9, loss_weights=[1.0, 1.0])))
    m.weights = om.init_weights(192, 10, 256, seed=1)
    tr = Trainer(m, bs, "cuda")
    planes, pol, val = vds.batch(env, idx)
    res["visit_targets_ms_512"] = event_ms(lambda: vds.visit_targets(lib, ids), 50)
    res["batch_ms_512"] = event_ms(lambda: vds.batch(env, idx), 20)
    res["train_step_ms_10x192_512"] = event_ms(lambda: tr.step_async(planes, pol, val, 1e-3), 20)
    res["visit_targets_share_of_step"] = res["visit_targets_ms_512"] / res["train_step_ms_10x192_512"]
    tr.close()
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
