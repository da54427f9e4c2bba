"""Time one SoundDetection request on the device: a 10 s 32 kHz clip (320 000 samples: 1001 frames; token grids
250 x 16, 125 x 8, 63 x 4, 32 x 2) through the shipped PVT, at B = 1 and B = 8.  Seeded synthetic weights
(specs.synth_pvt(PVT_SHIPPED)).  The engine and eager fp32 PyTorch (oracle/pvt_ref.py on the same GPU, TF32 off) are
alternated in one process; times are medians of CUDA-event intervals after warm-up.  Also prints the engine's launch
count per forward, its front end / transformer / head split (kernel time summed from one torch.profiler pass, in
launch order: the first three kernels are the front end, the last one the head), the FLOPs counted from the shapes,
and the GPU name and power limit read in the same run.

    python scripts/pvt_time.py [--reps 20]
"""
import argparse
import os
import re
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.audio_detection.audio_infer.pytorch.models import PVT  # noqa: E402
from oracle import pvt_ref as ref  # noqa: E402


def flops(cfg, n):
    """Multiply-adds x 2 per clip: the DFT GEMM, then per stage the patch embedding, q / kv / proj, sr conv, attention,
    fc1 / fc2 and the depthwise conv."""
    T = n // cfg["hop_size"] + 1
    fl = {"DFT": 2.0 * T * cfg["window_size"] * (cfg["window_size"] + 2), "patch": 0.0, "stages": []}
    cin = 1
    for i, (H, W) in enumerate(specs.pvt_grids(cfg, n)):
        C, sr, hid, N = cfg["embed_dims"][i], cfg["sr_ratios"][i], cfg["embed_dims"][i] * cfg["mlp_ratios"][i], H * W
        Nk = (H // sr) * (W // sr)
        fl["patch"] += 2.0 * N * C * cin * (49 if i == 0 else 9)
        blk = 2.0 * N * C * C * 2 + 2.0 * Nk * C * 2 * C + (2.0 * Nk * C * C * sr * sr if sr > 1 else 0.0)
        blk += 4.0 * N * Nk * C + 4.0 * N * C * hid + 2.0 * N * hid * 9
        fl["stages"].append(blk * cfg["depths"][i])
        cin = C
    return fl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pvt_time.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    cfg, n = specs.PVT_SHIPPED, 320000
    sd = specs.synth_pvt(cfg)
    m = PVT.from_config(cfg)
    m.load_state_dict(sd, strict=True)
    m = m.eval().to(dev)
    sdc = {k: v.to(dev) for k, v in sd.items()}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {q.stdout.strip()}")
    fl = flops(cfg, n)
    total = fl["DFT"] + fl["patch"] + sum(fl["stages"])
    print(f"FLOPs per 10 s clip: {total / 1e9:.2f} G (DFT {fl['DFT'] / 1e9:.2f}, patch embeddings {fl['patch'] / 1e9:.2f}, stages "
          + " / ".join(f"{s / 1e9:.2f}" for s in fl["stages"]) + ")")

    def timed(fns, reps):
        t = [[] for _ in fns]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for i in range(reps + 3):
            for k, f in enumerate(fns):        # alternated, so both arms see the same clocks and neighbours
                e0.record()
                f()
                e1.record()
                torch.cuda.synchronize()
                if i >= 3:
                    t[k].append(e0.elapsed_time(e1))
        return [statistics.median(x) for x in t]

    with torch.no_grad():
        for B in (1, 8):
            wav = torch.stack([specs.synth_pvt_wav(n, 40 + b) for b in range(B)]).to(dev)
            eng, eag = timed([lambda: m(wav, None), lambda: ref.forward(sdc, cfg, wav)], a.reps)
            base = _lib.launch_count()
            got = m(wav, None, return_logits=True)
            launches = _lib.launch_count() - base
            want = ref.forward(sdc, cfg, wav)
            err = ((got["logits"] - want["logits"]).double().pow(2).mean().sqrt() / want["logits"].double().pow(2).mean().sqrt()).item()
            print(f"B = {B}: engine {eng:7.2f} ms ({B * total / eng / 1e9:.2f} TFLOP/s, {launches} launches)   eager fp32 {eag:7.2f} ms   "
                  f"({eag / eng:.2f}x)   logits rel-RMSE engine vs eager {err:.2e}")
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
                m(wav, None)
                torch.cuda.synchronize()
            ks = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                         and "memset" not in e.name.lower()), key=lambda e: e.time_range.start)
            if len(ks) != launches:
                print(f"        stage split not available: the profiler recorded {len(ks)} kernels for {launches} launches")
                continue
            us = [e.device_time_total for e in ks]
            print(f"        kernel time: front end {sum(us[:3]) / 1e3:.3f} ms, transformer {sum(us[3:-1]) / 1e3:.3f} ms, "
                  f"head {us[-1] / 1e3:.3f} ms (sum {sum(us) / 1e3:.3f} ms of the {eng:.2f} ms request)")
            if B == 1:
                by = {}
                for e in ks:
                    hit = re.search(r"\w*kernel\w*", e.name)
                    nm = hit.group(0) if hit else e.name[:28]
                    c, t = by.get(nm, (0, 0.0))
                    by[nm] = (c + 1, t + e.device_time_total)
                for nm, (c, t) in sorted(by.items(), key=lambda kv: -kv[1][1]):
                    print(f"          {nm:28s} x{c:4d} {t / 1e3:8.3f} ms")


if __name__ == "__main__":
    main()
