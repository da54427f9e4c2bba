#!/usr/bin/env python
"""Time one TargetSoundDetection request on the engine against eager PyTorch.

One tool call: B = 1, a 10 s clip (T = 501 log-mel frames at 22.05 kHz, hop 441) and a 501-frame reference mel (a
stand-in: the shapes in ref_mel.pth are not in the reference tree), seeded weights at the shipped sizes with att_pool =
enhancement = True (the heaviest path).  The engine's stage times come from CUDA events it records at its stage
boundaries (agpt_tsd_stage_events); the eager arm is oracle/tsd_ref.py in fp32 with TF32 off, alternated with the engine
in the same process.  GFLOP are counted from the shapes (multiply-adds x 2; convs, Linears and the GRU).

    python scripts/tsd_time.py [--iters 20] [--warmup 3]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.audio_detection.target_sound_detection.src.models import RaDur_fusion  # noqa: E402
from oracle import tsd_ref as ref  # noqa: E402

STAGES = ("Cnn14(ref) + embedding", "Cnn14(x)", "features", "GRU pass 1", "enhance + GRU pass 2", "mix + interpolate")


def gflop(T, Tr):
    def cnn14(n):
        f, H, W, cin = 0, n, 64, 1
        for c, (ph, pw) in zip(specs.CNN14_CHANNELS, specs.TSD_ENC_POOLS):
            f += H * W * 9 * (cin * c + c * c)
            H, W, cin = H // ph, W // pw, c
        return f + H * 2048 * 128
    Td = specs.tsd_frames(specs.TSD_DEFAULT, T, Tr)[0]
    m = specs.tsd_stem_rows(T, 2)[3]
    pools = specs.TSD_POOLS[8]
    feat, H, W, cin = m * 32 * 96 * 2 * (1 + 9 + 25) // 2, m, 32, 96
    for c, (ph, pw) in zip(specs.TSD_DET_CHANNELS, pools[1:]):
        feat += H * W * 9 * (cin * c + c * c)
        H, W, cin = H // ph, W // pw, c
    feat += Td * 512 * 1024
    gru = Td * (512 * 3072 + 2 * 1536 * 512) + Td * 1024 * 2
    return {k: 2 * v / 1e9 for k, v in dict(ref=cnn14(Tr), x=cnn14(T), feat=feat, gru=gru).items()}


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
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = "cuda:0"
    cfg = specs.TSD_DEFAULT
    T = Tr = 501
    sd = specs.synth_tsd(cfg, 7171)
    m = RaDur_fusion(dict(att_pool=True, enhancement=True, tao=0.6, top=cfg["top"]), 64, 2, 125)
    m.load_state_dict(sd, strict=True)
    m = m.to(dev).eval()
    sdg = {k: v.to(dev) for k, v in sd.items()}
    x, r = specs.synth_tsd_mel(T, 1).to(dev), specs.synth_tsd_mel(Tr, 2).to(dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]
    for e in ev:
        e.record()
    torch.cuda.synchronize()
    m(x, r)
    arr = (C.c_void_p * len(ev))(*[e.cuda_event for e in ev])
    _lib.check(_lib.lib().agpt_tsd_stage_events(m._h, arr, len(ev)))

    def eager():
        with torch.no_grad():
            return ref.forward(sdg, cfg, x, r)

    for _ in range(a.warmup):
        m(x, r); eager()
    stage, whole, base = [], [], []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.iters):
        e0.record(); m(x, r); e1.record(); torch.cuda.synchronize()
        whole.append(e0.elapsed_time(e1))
        stage.append([ev[i].elapsed_time(ev[i + 1]) for i in range(len(STAGES))])
        e0.record(); eager(); e1.record(); torch.cuda.synchronize()
        base.append(e0.elapsed_time(e1))
    _lib.check(_lib.lib().agpt_tsd_stage_events(m._h, None, 0))
    d, up, _ = m(x, r)
    want = eager()
    g = gflop(T, Tr)
    st = np.median(np.array(stage), axis=0)
    print(f"GPU: {torch.cuda.get_device_name(0)}, power limit {power_limit()}")
    print(f"one request: B = 1, T = {T}, Tr = {Tr}, att_pool = enhancement = True, top = {cfg['top']}; "
          f"medians of {a.iters} alternated runs (ms)")
    flops = [g["ref"], g["x"], g["feat"], g["gru"], g["gru"], 0.0]
    for name, t, f in zip(STAGES, st, flops):
        print(f"  {name:<24s} {t:8.3f} ms" + (f"   {f:6.2f} GFLOP  {f / t:6.2f} TFLOP/s" if f else ""))
    tot = sum(flops)
    print(f"  {'whole call (engine)':<24s} {np.median(whole):8.3f} ms   {tot:6.2f} GFLOP  {tot / np.median(whole):6.2f} TFLOP/s")
    print(f"  {'eager fp32 (oracle)':<24s} {np.median(base):8.3f} ms   speed-up {np.median(base) / np.median(whole):.2f}x")
    print(f"  decision_up max-abs vs eager fp32: {(up - want['decision_up']).abs().max().item():.2e}")


if __name__ == "__main__":
    main()
