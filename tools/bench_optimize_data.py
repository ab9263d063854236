"""OptimizeWorker's play data on one GPU: `fill_queue` wall time on the host path (records.expanding_data: one replay
launch per ply, planes copied back per game, one-hot rows built in Python) against the device path (the files packed on
the host, one cz_play_replay launch), alternated in one process; bytes per position of both datasets; and one device
batch's assembly (gather, cz_env_encode_planes, one-hot scatter; 14 and 28 planes) against one cz_train_step.

    python tools/bench_optimize_data.py [--files 100] [--games-per-file 5] [--fills 4] [--reps 3]

The records are seeded engine self-play games (random 64x2 net, 8 simulations per move, max_game_length 100 as in
configs/normal.py, no resignation), written as play-data files of `--games-per-file` games.  Everything it writes goes
to a temporary directory.
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
from cczero_b200.env import StaticEnv  # noqa: E402
from cczero_b200.lib import get_lib  # noqa: E402
from oracle import model as om  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit not readable"


def selfplay_records(lib, n_games, seed, max_game_length=100):
    from cczero_b200.engine import Engine
    w = om.init_weights(64, 2, 256, seed=seed)
    eng = Engine(lib, "cuda", n_games=n_games, sims_per_move=8, leaves_per_round=4, nn_filters=64, nn_blocks=2,
                 max_game_length=max_game_length, seed=seed, enable_resign_rate=0.0)
    eng.set_weights({k: torch.as_tensor(v) for k, v in w.items()})
    eng.reset()
    recs = []
    while len(recs) < n_games:
        eng.selfplay(target_games=n_games - len(recs), max_moves=0)
        recs += eng.drain_records()
    eng.close()
    return [rd.record_to_play_data(r) for r in sorted(recs, key=lambda r: r["game_index"])[:n_games]]


def worker(env, path, history):
    from cczero_b200.optimize import OptimizeWorker
    tc = SimpleNamespace(dataset_size=10 ** 9, batch_size=512)
    cfg = SimpleNamespace(trainer=tc, opts=SimpleNamespace(has_history=history))
    return OptimizeWorker(cfg, env=env, device="cuda", dataset=path)


def time_fill(env, file_sets, path, history, seed):
    """Wall time of one fill_queue per set of files (the dataset grows across them, as when it carries over)."""
    w = worker(env, path, history)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for files in file_sets:
        w.filenames = deque(files)
        Random(seed).shuffle(w.filenames)
        w.fill_queue()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, w


def event_ms(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def time_batches(lib, env, ds, filters, blocks, bs, reps=20):
    from cczero_b200.model import CChessModel
    from cczero_b200.train import Trainer
    out = {}
    idx = np.random.RandomState(0).permutation(len(ds))[:bs]
    for history in (False, True):
        planes_n = 28 if history else 14
        out[f"batch_ms_{planes_n}"] = event_ms(lambda: ds.batch(env, idx, history), reps)
        mc = SimpleNamespace(cnn_filter_num=filters, res_layer_num=blocks, value_fc_size=256, l2_reg=1e-4,
                             input_depth=planes_n, policy_channels=4, value_channels=2, cnn_first_filter_size=5,
                             cnn_filter_size=3)
        m = CChessModel(SimpleNamespace(model=mc, trainer=SimpleNamespace(momentum=0.9, loss_weights=[1.0, 1.0])))
        m.weights = om.init_weights(filters, blocks, 256, seed=1, in_planes=planes_n)
        tr = Trainer(m, bs, "cuda")
        planes, pol, val = ds.batch(env, idx, history)
        out[f"train_step_ms_{planes_n}"] = event_ms(lambda: tr.step_async(planes, pol, val, 1e-3), reps)
        out[f"batch_share_of_step_{planes_n}"] = out[f"batch_ms_{planes_n}"] / out[f"train_step_ms_{planes_n}"]
        tr.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=100, help="files per fill_queue (configs/normal.py load_data_steps)")
    ap.add_argument("--games-per-file", type=int, default=5, help="nb_game_in_file")
    ap.add_argument("--fills", type=int, default=4, help="fill_queue calls per timed run, each on its own files")
    ap.add_argument("--reps", type=int, default=3, help="alternated host / device fills")
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    lib = get_lib()
    env = StaticEnv(lib, "cuda")
    res = {"card": card()}
    print(json.dumps(res), flush=True)
    n_games = args.files * args.games_per_file * args.fills
    t0 = time.perf_counter()
    recs = selfplay_records(lib, n_games, args.seed)
    plies = np.array([len(r) - 1 for r in recs])
    res["records"] = {"games": n_games, "positions": int(plies.sum()), "mean_plies": float(plies.mean()),
                      "selfplay_s": time.perf_counter() - t0}
    print(json.dumps({"records": res["records"]}), flush=True)
    with tempfile.TemporaryDirectory() as d:
        files = []
        for i in range(args.files * args.fills):
            p = os.path.join(d, f"play_{i:05d}.json")
            with open(p, "w") as f:
                json.dump(sum(recs[i * args.games_per_file:(i + 1) * args.games_per_file], []), f)
            files.append(p)
        sets = [files[k * args.files:(k + 1) * args.files] for k in range(args.fills)]
        for history in (False, True):
            key = f"fill_queue_{28 if history else 14}"
            times = {"host": [], "device": []}
            time_fill(env, [files[:2]], "host", history, 0)             # warm both paths
            time_fill(env, [files[:2]], "device", history, 0)
            for r in range(args.reps):
                for path in (("host", "device") if r % 2 == 0 else ("device", "host")):
                    t, w = time_fill(env, sets, path, history, r)
                    times[path].append(t)
                    n = w.loaded_count()
                    if path == "host":
                        host_bytes = sum(np.asarray(w.dataset[i][0]).nbytes for i in range(3))
                    else:
                        ds = w.dataset
                        dev_bytes = sum(x.numel() * x.element_size() for x in (ds.boards, ds.labels, ds.values, ds.ply)) / n
            res[key] = {"positions": n, "fill_queue_calls": args.fills, "host_s": times["host"], "device_s": times["device"],
                        "host_positions_per_s": n / min(times["host"]), "device_positions_per_s": n / min(times["device"]),
                        "speedup": min(times["host"]) / min(times["device"]),
                        "host_array_bytes_per_position": host_bytes, "device_bytes_per_position": dev_bytes}
            print(json.dumps({key: res[key]}), flush=True)
    for f, b, bs in ((192, 10, 512), (256, 20, 1024)):
        key = f"batch_vs_step_{f}x{b}@{bs}"
        res[key] = time_batches(lib, env, ds, f, b, bs)
        print(json.dumps({key: res[key]}), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
