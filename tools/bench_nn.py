"""Micro-benchmarks of the network kernels on one GPU (development aid; bench.py is the contract)."""
import ctypes as C
import sys
import os
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from cczero_b200.lib import get_lib
from cczero_b200.engine import Engine
from oracle import model as om


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def time_it(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    lib = get_lib()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    # the product kernel: wgmma conv on dense activations (im2col TMA), without / with the fp16 skip stream
    for c, nb in ((256, 8192), (256, 4096), (128, 2048), (128, 8192), (192, 4096)):
        x = torch.randn(nb, 10, 9, c, device="cuda").half()
        w = (torch.randn(9, c, c, device="cuda") * 0.02).half()
        b = torch.zeros(c, device="cuda")
        y = torch.empty_like(x)
        for res, tag in ((None, "no skip"), (x, "fp16 skip")):
            ms = time_it(lambda: lib.call("cz_igemm_conv3x3_dense", p(x), p(w), p(b), p(res), p(y), nb, c, 1, st))
            fl = 2.0 * nb * 90 * 9 * c * c
            print(f"conv3x3 dense C={c} boards={nb} {tag}: {ms * 1e3:.1f} us  {fl / ms / 1e9:.1f} TFLOP/s")
    for (f, bl, batch) in ((128, 7, 2048), (256, 20, 8192), (256, 20, 1024), (256, 20, 4096)):
        eng = Engine(lib, "cuda", n_games=batch, sims_per_move=8, leaves_per_round=1, nn_filters=f, nn_blocks=bl)
        w = om.init_weights(f, bl, 256, seed=0)
        eng.set_weights({k: torch.as_tensor(v) for k, v in w.items()})
        boards = torch.zeros(batch, 96, dtype=torch.uint8, device="cuda")
        from cczero_b200.env import state_to_board
        from oracle import senv
        boards[:] = torch.as_tensor(state_to_board(senv.INIT_STATE)).cuda()
        ms = time_it(lambda: eng.nn_forward_boards(boards), iters=5, warm=2)
        flops = 2 * 90 * (350 * f + bl * 18 * f * f + 6 * f) + 2 * (360 * 2086 + 180 * 256 + 256)
        print(f"forward {f}x{bl} batch={batch}: {ms:.2f} ms  {batch / ms * 1e3:.0f} pos/s  {batch * flops / ms / 1e9:.1f} TFLOP/s")
        eng.close()


if __name__ == "__main__":
    main()
