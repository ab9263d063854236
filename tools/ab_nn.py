"""Interleaved A/B of the network forward under different kernel selections (environment variables read at engine creation).
Every variant runs in its own subprocess, round-robin over `rounds`, each measurement a multi-second back-to-back loop so that
the part sits at its power-cap equilibrium; medians are reported.  python tools/ab_nn.py [rounds]"""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = {
    "default": {},
    "no programmatic dependent launch": {"CZ_PDL": "0"},
    "no 64-column tiles for small batches": {"CZ_NSPLIT": "0"},
    "skip fp16 only (upper bound: breaks 1e-3 at 20 blocks)": {"CZ_FP32_SKIP": "0"},
}
SHAPES = [(256, 20, 8192, 3.0), (128, 7, 2048, 1.5), (192, 10, 4096, 1.5)]
if os.environ.get("AB_ONLY"):                      # e.g. AB_ONLY="default,no programmatic" AB_SHAPES=small
    keep = [k.strip() for k in os.environ["AB_ONLY"].split(",")]
    VARIANTS = {k: v for k, v in VARIANTS.items() if any(k.startswith(p) for p in keep)}
if os.environ.get("AB_SHAPES") == "c3":
    SHAPES = [(256, 20, 8192, 3.0)]
if os.environ.get("AB_SHAPES") == "small":
    SHAPES = [(128, 7, 2048, 1.5), (128, 7, 8192, 1.5), (64, 4, 2048, 1.0)]

CHILD = r'''
import sys, time, json, torch
sys.path.insert(0, %r)
from cczero_b200.engine import Engine
from cczero_b200.lib import get_lib
from cczero_b200.env import state_to_board
from oracle import model as om, senv
out = {}
for f, bl, batch, secs in %r:
    eng = Engine(get_lib(), "cuda", n_games=batch, sims_per_move=8, leaves_per_round=1, nn_filters=f, nn_blocks=bl)
    eng.set_weights({k: torch.as_tensor(v) for k, v in om.init_weights(f, bl, 256, seed=0).items()})
    boards = torch.zeros(batch, 96, dtype=torch.uint8, device="cuda")
    boards[:] = torch.as_tensor(state_to_board(senv.INIT_STATE)).cuda()
    for _ in range(3):
        eng.nn_forward_boards(boards)
    torch.cuda.synchronize()
    t0 = time.perf_counter(); n = 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    while time.perf_counter() - t0 < secs:
        for _ in range(4):
            eng.nn_forward_boards(boards)
        n += 4
        torch.cuda.synchronize()
    e1.record(); torch.cuda.synchronize()
    out["%%dx%%d@%%d" %% (f, bl, batch)] = e0.elapsed_time(e1) / n
    eng.close()
print(json.dumps(out))
'''


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    res = {k: {} for k in VARIANTS}
    for r in range(rounds):
        for name, env in VARIANTS.items():
            e = dict(os.environ, **env)
            p = subprocess.run([sys.executable, "-c", CHILD % (ROOT, SHAPES)], env=e, capture_output=True, text=True, timeout=600)
            line = [l for l in p.stdout.splitlines() if l.startswith("{")]
            if not line:
                print(name, "FAILED", p.stderr[-400:])
                continue
            for k, v in json.loads(line[-1]).items():
                res[name].setdefault(k, []).append(v)
    for name, d in res.items():
        print(name, {k: round(statistics.median(v), 3) for k, v in d.items()}, {k: [round(x, 3) for x in v] for k, v in d.items()})


if __name__ == "__main__":
    main()
