#!/usr/bin/env python
"""Time one Binaural tool request on the engine against the reference's eager per-chunk loop.

One tool call: a 10 s mono clip at 48 kHz (480000 samples, 1200 view frames), seeded weights at the shipped size (4 x
64) and a seeded trajectory.  The engine arm is BinauralNetwork.binauralize (every chunk and ear in one call); the eager
arm is oracle/binaural_ref.py's chunk loop on the same GPU with TF32 off and the quaternion rotation on the host, as the
reference does it (one device synchronisation per chunk).  The two are alternated in one process and timed with CUDA
events; launches are the engine's own count (agpt_launch_count) per call.

    python scripts/binaural_time.py [--iters 20] [--warmup 3]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.mono2binaural.src.models import BinauralNetwork  # noqa: E402
from oracle import binaural_ref as ref  # noqa: E402


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=20).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seconds", type=int, default=10)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = "cuda:0"
    L = 48000 * a.seconds
    sd = specs.synth_binaural(specs.BINAURAL, 4242)
    net = BinauralNetwork()
    net.load_state_dict(sd, strict=True)
    net.eval()
    sdg = {k: v.to(dev) for k, v in sd.items()}
    mono = specs.synth_binaural_mono(L, 1).to(dev)
    view = specs.synth_binaural_view(L // 400, 2)[0].to(dev)

    def engine():
        return net.binauralize(mono, view)

    def eager():
        return ref.tool(mono, view, lambda m, v: ref.forward(sdg, specs.BINAURAL, m, v, host_rotation=True))

    for _ in range(a.warmup):
        engine(); eager()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    eng, base, launches = [], [], []
    for _ in range(a.iters):
        n0 = _lib.launch_count()
        e0.record(); engine(); e1.record(); torch.cuda.synchronize()
        eng.append(e0.elapsed_time(e1))
        launches.append(_lib.launch_count() - n0)
        e0.record(); eager(); e1.record(); torch.cuda.synchronize()
        base.append(e0.elapsed_time(e1))
    y, want = engine(), eager()
    rows = len(specs.binaural_chunks(L, L // 400)[1])
    print(f"GPU: {torch.cuda.get_device_name(0)}, power limit {power_limit()}")
    print(f"one request: {a.seconds} s at 48 kHz ({L} samples, {rows} chunks); medians of {a.iters} alternated runs")
    print(f"  engine binauralize        {np.median(eng) * 1e3:9.1f} us   ({np.min(eng) * 1e3:.1f} min)   launches per call {max(launches)}")
    print(f"  eager per-chunk loop      {np.median(base) * 1e3:9.1f} us   ({np.min(base) * 1e3:.1f} min)   "
          f"speed-up {np.median(base) / np.median(eng):.1f}x")
    print(f"  max-abs engine vs eager: {(y - want).abs().max().item():.2e}")


if __name__ == "__main__":
    main()
