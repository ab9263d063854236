"""Where the residual conv's time goes: conv1 (x -> t, fp16 out) against conv2 (t + skip -> y, fp16 + fp32 skip copy out).

Runs nn_forward_boards on seeded random-init weights under torch.profiler (CUDA activities) and reports the median duration
of the tower's k_igemm launches, split into conv1 (1st, 3rd, ... launch of a forward) and conv2 (2nd, 4th, ...).  Both convs
do the same MMAs; conv2's epilogue additionally reads the skip stream and writes its fp32 copy.  Run at batch 8192 (the
activations stream from HBM) and at batch 1024 (they stay in L2), so a gap that is the epilogue's HBM traffic shows up as
conv2 > conv1 at 8192 and shrinks at 1024.

Each row also carries the MMA-only lower bound of a launch at the sampled median SM clock, from shapes alone: the waves of
M x N tiles over the SMs times 2 * M * N * 9C FLOP per tile, at 4096 dense fp16 FLOP per clock per SM.  What a tile takes
beyond that bound is conv1's main-loop plus epilogue loss; what conv2 takes beyond conv1 is its epilogue's.  Beside it, the
operand bytes a tile's main loop moves from L2 to shared memory: the tile's input rows with their halo once per 64-channel
block, and the weights' N tile for every tap and block.

    python tools/bench_conv_epilogue.py [--filters 256] [--blocks 20] [--batches 8192,1024] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from cczero_b200.engine import Engine
from cczero_b200.env import state_to_board
from cczero_b200.lib import get_lib
from oracle import model as om
from oracle import senv

HALO_BOX = 152                  # rows per TMA box of the conv's A operand (csrc/cz_igemm.cuh kHaloBox)
SM_FLOP_PER_CLK = 4096          # dense fp16 tensor-core FLOP per clock per SM (H100 data sheet: 989 TFLOP/s, 132 SMs, 1830 MHz)


def smi(fields):
    p = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={fields}", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return p.stdout.strip()


def conv_tile(c, batch, sms):
    """M x N tile of the full-width conv (cznn::conv_args): N = 128 at C = 256, else C; M = 256 when those tiles fill at
    least 8 waves and C != 192, else 128."""
    n = 128 if c == 256 else c
    m = 256 if c != 192 and (batch * 90 + 255) // 256 * (c // n) >= 8 * sms else 128
    return m, n


def operand_bytes(c, m, n):
    """L2 -> shared memory bytes of one tile's main loop: A = M / 128 halo boxes per 64-channel block, B = 9 taps x C / 64
    blocks of N x 64 fp16 weights."""
    return {"a": (m // 128) * HALO_BOX * 128 * (c // 64), "b": 9 * (c // 64) * n * 128}


def shape_bytes(c, m, n, fp32_skip):
    """HBM bytes per M x N tile, from shapes: the tile's own input pixels (the 3x3 halo and the weights are L2 hits), the
    skip it reads and what it writes."""
    a = m * c * 2
    conv1 = {"operand": a, "epilogue_read": 0, "epilogue_write": m * n * 2}
    skip = m * n * (4 if fp32_skip else 2)
    conv2 = {"operand": a, "epilogue_read": skip, "epilogue_write": m * n * 2 + (m * n * 4 if fp32_skip else 0)}
    return conv1, conv2


def measure(lib, filters, blocks, batch, forwards, seed):
    eng = Engine(lib, "cuda", n_games=batch, sims_per_move=8, leaves_per_round=1, nn_filters=filters, nn_blocks=blocks)
    eng.set_weights({k: torch.as_tensor(v) for k, v in om.init_weights(filters, blocks, 256, seed=seed).items()})
    boards = torch.zeros(batch, 96, dtype=torch.uint8, device="cuda")
    boards[:] = torch.as_tensor(state_to_board(senv.INIT_STATE)).cuda()
    for _ in range(3):
        eng.nn_forward_boards(boards)
    torch.cuda.synchronize()
    sampler = subprocess.Popen(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                                "-lms", "100"], stdout=subprocess.PIPE, text=True)
    try:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(forwards):
                eng.nn_forward_boards(boards)
            torch.cuda.synchronize()
    finally:
        sampler.terminate()
        clk_out, _ = sampler.communicate(timeout=30)
    eng.close()
    clocks = [int(x) for x in clk_out.split() if x.strip().isdigit()]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tm, tn = conv_tile(filters, batch, sms)
    name = f"k_igemm<{tn}, {tm}, true>"            # the tower's convs; the policy GEMM is k_igemm<256, 128, false>
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and name in e.name),
                key=lambda e: e.time_range.start)
    per_fwd = 2 * blocks
    assert len(ev) == forwards * per_fwd, (len(ev), forwards, per_fwd)
    us1, us2 = [], []
    for f in range(forwards):
        tower = ev[f * per_fwd: f * per_fwd + 2 * blocks]
        us1 += [e.time_range.elapsed_us() for e in tower[0::2]]
        us2 += [e.time_range.elapsed_us() for e in tower[1::2]]
    flop = 2.0 * batch * 90 * 9 * filters * filters
    tiles = (batch * 90 + tm - 1) // tm * (filters // tn)
    b1, b2 = shape_bytes(filters, tm, tn, blocks >= 10)
    row = {"filters": filters, "blocks": blocks, "batch": batch, "tile": f"{tm}x{tn}", "tiles": tiles,
           "l2_to_smem_bytes_per_tile": operand_bytes(filters, tm, tn)}
    for tag, us, b in (("conv1", us1, b1), ("conv2", us2, b2)):
        med = statistics.median(us)
        row[tag] = {"median_us": round(med, 1), "min_us": round(min(us), 1), "max_us": round(max(us), 1), "launches": len(us),
                    "tflops": round(flop / med / 1e6, 1), "hbm_bytes_per_tile": b, "hbm_gb_s": round(tiles * sum(b.values()) / med / 1e3, 1)}
    row["conv2_over_conv1"] = round(row["conv2"]["median_us"] / row["conv1"]["median_us"], 3)
    row["sm_clock_mhz"] = {"median": statistics.median(clocks) if clocks else None, "min": min(clocks, default=None),
                           "max": max(clocks, default=None), "samples": len(clocks)}
    if clocks:
        waves = (tiles + sms - 1) // sms
        tile_us = 2.0 * tm * tn * 9 * filters / (SM_FLOP_PER_CLK * row["sm_clock_mhz"]["median"])
        row["mma_bound"] = {"waves": waves, "tile_us": round(tile_us, 2), "launch_us": round(waves * tile_us, 1)}
        for tag in ("conv1", "conv2"):
            row[tag]["tile_excess_us"] = round(row[tag]["median_us"] / waves - tile_us, 2)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--filters", type=int, default=256)
    ap.add_argument("--blocks", type=int, default=20)
    ap.add_argument("--batches", default="8192,1024")
    ap.add_argument("--forwards", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="also write the result as JSON into this directory")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    lib = get_lib()
    card = smi("name,power.limit,clocks.max.sm")
    rows = [measure(lib, args.filters, args.blocks, int(b), args.forwards, args.seed) for b in args.batches.split(",")]
    res = {"card": card, "rows": rows}
    for r in rows:
        print(f"{r['filters']}x{r['blocks']} batch {r['batch']} ({r['tiles']} tiles of {r['tile']})  SM clock {r['sm_clock_mhz']['median']} MHz")
        for tag in ("conv1", "conv2"):
            c = r[tag]
            print(f"  {tag}: {c['median_us']:8.1f} us median [{c['min_us']}, {c['max_us']}] over {c['launches']}  {c['tflops']:6.1f} TFLOP/s"
                  f"  HBM bytes/tile {c['hbm_bytes_per_tile']}  ({c['hbm_gb_s']} GB/s)")
        print(f"  conv2 / conv1 = {r['conv2_over_conv1']}")
        if "mma_bound" in r:
            b = r["mma_bound"]
            print(f"  MMA-only bound at that clock: {b['launch_us']} us per launch ({b['waves']} waves x {b['tile_us']} us per tile);"
                  f" per-tile excess conv1 {r['conv1']['tile_excess_us']} us, conv2 {r['conv2']['tile_excess_us']} us")
        ob = r["l2_to_smem_bytes_per_tile"]
        print(f"  L2 -> shared operand bytes per tile: A {ob['a']}, B {ob['b']}, total {ob['a'] + ob['b']}")
    print("card, power limit, max SM clock:", card)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "conv_epilogue.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
