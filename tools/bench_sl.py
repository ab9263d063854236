"""Supervised-learning throughput on one GPU: cz_sl_replay on seeded synthetic games (against the pure-Python light-board
replay of the same games on the host), cz_train_step with SGD against Adam, the fused Adam launch alone, and the bytes
per position of the device dataset against the reference's host arrays.

    python tools/bench_sl.py
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cczero_b200  # noqa: E402,F401
from cczero_b200 import sl_data as sd  # noqa: E402
from cczero_b200.lib import get_lib  # noqa: E402
from oracle import model as om  # noqa: E402
from oracle import senv as osenv  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception:
        out = torch.cuda.get_device_name(0) + ", power limit not readable"
    return out


def synthetic(n, seed):
    """Seeded legal playouts as onegreen digit moves (every move resolves, so whole games replay)."""
    rng = np.random.RandomState(seed)
    games, host = [], []
    for _ in range(n):
        s, plies, sides, moves = osenv.INIT_STATE, [], [], []
        red = True
        for k in range(rng.randint(60, 140)):
            lm = osenv.get_legal_moves(s)
            if not lm or osenv.done(s)[0]:
                break
            m = lm[rng.randint(len(lm))]
            a = m if red else osenv.flip_move(m)                 # the light board's frame
            plies.append(f"{a[0]}{9 - int(a[1])}{a[2]}{9 - int(a[3])}".encode())
            sides.append(1 if red else -1)
            moves.append(a)
            s = osenv.step(s, m)
            red = not red
        games.append((plies, sides))
        host.append(moves)
    return games, host


def python_replay(moves_per_game):
    """The reference's per-ply host work, restated: light-board push and the observation string per ply."""
    t0 = time.perf_counter()
    for moves in moves_per_game:
        b = [list(r) for r in ("rnbakabnr", ".........", ".c.....c.", "p.p.p.p.p", ".........", ".........",
                               "P.P.P.P.P", ".C.....C.", ".........", "RNBAKABNR")]
        red = True
        for a in moves:
            x0, y0, x1, y1 = (int(c) for c in a)
            rows = b if red else [r[::-1] for r in b[::-1]]
            "/".join("".join(r) for r in rows[::-1])
            b[y1][x1] = b[y0][x0]
            b[y0][x0] = '.'
            red = not red
    return time.perf_counter() - t0


def time_replay(lib, games, reps=5):
    b0 = np.stack([sd.start_board()] * len(games))
    plies, sides = [p for p, _ in games], [s for _, s in games]
    sd.replay(lib, "cuda", b0, plies, sides, sd.ONEGREEN)
    torch.cuda.synchronize()
    # the kernel alone: inputs staged once, timed with CUDA events
    rep = sd.replay(lib, "cuda", b0, plies, sides, sd.ONEGREEN)
    assert (rep.status == sd.OK).all()
    npos = int(rep.offsets[-1])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        sd.replay(lib, "cuda", b0, plies, sides, sd.ONEGREEN)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return npos, min(ts)


def time_train(lib, filters, blocks, bs, steps=10):
    from types import SimpleNamespace
    from cczero_b200.model import CChessModel
    from cczero_b200.train import Trainer
    mc = SimpleNamespace(cnn_filter_num=filters, res_layer_num=blocks, value_fc_size=256, l2_reg=1e-4, input_depth=14,
                         policy_channels=4, value_channels=2, cnn_first_filter_size=5, cnn_filter_size=3)
    cfg = SimpleNamespace(model=mc, trainer=SimpleNamespace(momentum=0.9, loss_weights=[1.0, 1.0]))
    m = CChessModel(cfg)
    m.weights = om.init_weights(filters, blocks, 256, seed=1)
    rng = np.random.RandomState(0)
    planes = torch.zeros((bs, 14, 10, 9), device="cuda")
    planes[:, 0, 0, :] = 1
    pol = torch.zeros((bs, om.N_LABELS), device="cuda")
    pol[torch.arange(bs), torch.as_tensor(rng.randint(0, om.N_LABELS, bs))] = 1
    val = torch.as_tensor(rng.choice([-1.0, 1.0], bs).astype(np.float32), device="cuda")
    out = {}
    for opt in ("sgd", "adam"):
        tr = Trainer(m, bs, "cuda", optimizer=opt)
        for _ in range(3):
            tr.step_async(planes, pol, val, 1e-3)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            tr.step_async(planes, pol, val, 1e-3)
        e1.record()
        torch.cuda.synchronize()
        out[opt + "_step_ms"] = e0.elapsed_time(e1) / steps
        if opt == "adam":
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(steps):
                    tr.step_async(planes, pol, val, 1e-3)
                torch.cuda.synchronize()
            ev = [e for e in prof.key_averages() if "k_adam" in e.key]
            out["adam_launch_us"] = (ev[0].device_time_total / ev[0].count) if ev else None
            out["adam_launches_per_step"] = (ev[0].count / steps) if ev else None
        tr.close()
    return out


def main():
    lib = get_lib()
    res = {"card": card()}
    base, base_host = synthetic(2000, seed=1)
    for n in (2000, 20000):
        games, host = base * (n // 2000), base_host * (n // 2000)      # 20 000 = the 2 000 seeded games ten times
        npos, t = time_replay(lib, games)
        th = python_replay(host)
        res[f"replay_{n}"] = {"games_per_s": n / t, "positions_per_s": npos / t, "positions": npos, "seconds": t,
                              "python_host_seconds": th}
        print(json.dumps({f"replay_{n}": res[f"replay_{n}"]}), flush=True)
    for f, b, bs in ((192, 10, 512), (256, 20, 1024)):
        res[f"train_{f}x{b}@{bs}"] = time_train(lib, f, b, bs)
        print(json.dumps({f"train_{f}x{b}@{bs}": res[f"train_{f}x{b}@{bs}"]}), flush=True)
    ref_bytes = 14 * 90 * 4 + om.N_LABELS * 4 + 4
    res["bytes_per_position"] = {"device_dataset": 96 + 2 + 4, "reference_host_arrays": ref_bytes}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
