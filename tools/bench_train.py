"""Training throughput of cz_train_step against the PyTorch step a user would otherwise write (fp16 autocast,
channels_last, cuDNN), on the same network and batch.

    python tools/bench_train.py [--steps 10] [--warmup 3] [--configs 256x7@512,192x10@1024,256x20@1024]

Per configuration: training positions/s over a warmed window timed with CUDA events; TFLOP/s of the forward 3x3 convs,
the dgrad convs (both igemm::k_igemm: the first 2*blocks launches of a step are the forward, the next 2*blocks the
dgrad) and wgrad::k_wgrad, from torch.profiler kernel times, each at 2*90*9*C^2 algorithmic FLOPs per conv per position;
and the PyTorch baseline's positions/s.  Prints the card name and power limit with the numbers.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import model as om  # noqa: E402


def random_batch(n, seed=0):
    rng = np.random.RandomState(seed)
    planes = np.zeros((n, 14, 10, 9), np.float32)
    occ = rng.rand(n, 90) < 0.35
    piece = rng.randint(0, 14, (n, 90))
    b, pix = np.nonzero(occ)
    planes[b, piece[b, pix], pix // 9, pix % 9] = 1
    pol = np.zeros((n, om.N_LABELS), np.float32)
    pol[np.arange(n), rng.randint(0, om.N_LABELS, n)] = 1
    return planes, pol, rng.choice([-1.0, 0.0, 1.0], n).astype(np.float32)


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return out or None
    except Exception:
        return None


def bench_cuda(filters, blocks, n, steps, warmup):
    from cczero_b200.model import CChessModel
    from cczero_b200.train import Trainer
    mc = SimpleNamespace(cnn_filter_num=filters, res_layer_num=blocks, value_fc_size=256, l2_reg=1e-4, input_depth=14)
    cfg = SimpleNamespace(model=mc, trainer=SimpleNamespace(momentum=0.9, loss_weights=[1.0, 1.0]))
    m = CChessModel(cfg).build(seed=0)
    tr = Trainer(m, n, "cuda")
    planes, pol, val = (torch.as_tensor(x, device="cuda") for x in random_batch(n))
    for _ in range(warmup):
        tr.step_async(planes, pol, val, 0.01)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        tr.step_async(planes, pol, val, 0.01)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tr.step_async(planes, pol, val, 0.01)
        torch.cuda.synchronize()
    ev = sorted([e for e in prof.events() if e.device_type.name == "CUDA"], key=lambda e: e.time_range.start)
    igemm = [e.time_range.elapsed_us() for e in ev if "k_igemm" in e.name]
    wgrad = [e.time_range.elapsed_us() for e in ev if "k_wgrad<" in e.name or "k_wgradILi" in e.name]
    conv_flops = 2.0 * 90 * 9 * filters * filters * n
    nc = 2 * blocks
    tf = lambda us, k: (conv_flops * k / (sum(us) * 1e-6) / 1e12) if us and sum(us) > 0 else None
    tr.close()
    return {"positions_per_s": n / (ms * 1e-3), "step_ms": ms, "fwd_conv_tflops": tf(igemm[:nc], nc),
            "dgrad_tflops": tf(igemm[nc:2 * nc], nc), "wgrad_tflops": tf(wgrad, len(wgrad)),
            "fwd_conv_ms": sum(igemm[:nc]) / 1e3, "dgrad_ms": sum(igemm[nc:2 * nc]) / 1e3, "wgrad_ms": sum(wgrad) / 1e3}


class TorchNet(nn.Module):
    """agent/model.py's network in PyTorch (BN eps 1e-3, momentum 0.01 = Keras 0.99)."""

    def __init__(self, c, blocks, pol_c=4, val_c=2, fc=256):
        super().__init__()
        bn = lambda k: nn.BatchNorm2d(k, eps=1e-3, momentum=0.01)
        self.first = nn.Sequential(nn.Conv2d(14, c, 5, padding=2, bias=False), bn(c), nn.ReLU())
        self.blocks = nn.ModuleList(nn.ModuleList([nn.Conv2d(c, c, 3, padding=1, bias=False), bn(c),
                                                   nn.Conv2d(c, c, 3, padding=1, bias=False), bn(c)]) for _ in range(blocks))
        self.pol = nn.Sequential(nn.Conv2d(c, pol_c, 1, bias=False), bn(pol_c), nn.ReLU(), nn.Flatten(), nn.Linear(pol_c * 90, om.N_LABELS))
        self.val = nn.Sequential(nn.Conv2d(c, val_c, 1, bias=False), bn(val_c), nn.ReLU(), nn.Flatten(), nn.Linear(val_c * 90, fc),
                                 nn.ReLU(), nn.Linear(fc, 1), nn.Tanh())

    def forward(self, x):
        x = self.first(x)
        for c1, b1, c2, b2 in self.blocks:
            x = F.relu(x + b2(c2(F.relu(b1(c1(x))))))
        return self.pol(x), self.val(x)[:, 0]


def bench_torch(filters, blocks, n, steps, warmup):
    torch.backends.cudnn.benchmark = True
    net = TorchNet(filters, blocks).cuda().to(memory_format=torch.channels_last)
    opt = torch.optim.SGD(net.parameters(), lr=0.01, momentum=0.9, weight_decay=0.0)
    planes, pol, val = (torch.as_tensor(x, device="cuda") for x in random_batch(n))
    planes = planes.contiguous(memory_format=torch.channels_last)
    scaler = torch.amp.GradScaler("cuda")

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            logits, v = net(planes)
            loss = F.cross_entropy(logits.float(), pol.argmax(1)) + F.mse_loss(v.float(), val)
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return {"positions_per_s": n / (ms * 1e-3), "step_ms": ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", default="256x7@512,192x10@1024,256x20@1024")
    a = ap.parse_args()
    dev = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    print(json.dumps(dev))
    for spec in a.configs.split(","):
        fb, n = spec.split("@")
        f, b = (int(x) for x in fb.split("x"))
        res = {"config": spec, **dev, "cuda": bench_cuda(f, b, int(n), a.steps, a.warmup), "pytorch": bench_torch(f, b, int(n), a.steps, a.warmup)}
        res["speedup_vs_pytorch"] = res["cuda"]["positions_per_s"] / res["pytorch"]["positions_per_s"]
        print(json.dumps(res))


if __name__ == "__main__":
    main()
