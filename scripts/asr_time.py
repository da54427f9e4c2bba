"""Time the ASR call of one TTS_OOD request on the device: Wav2Vec2ForCTC (base-960h config, seeded weights from
specs.synth_w2v) on a 3, 10 and 20 s reference clip at 16 kHz, B = 1.  The engine and transformers' eager
Wav2Vec2ForCTC (fp32, TF32 off, the same GPU) are alternated in one process after every length has been warmed up;
times are medians of CUDA-event intervals.  Also prints the FLOPs counted from the shapes, the engine's launches per
call, the sum of its kernels' device time in one torch.profiler pass (the rest of the call is host work and launch
gaps), the logits' rel-RMSE between the two arms, and the GPU name and power limit read in the same run.

    python scripts/asr_time.py [--reps 20]
"""
import argparse
import os
import re
import statistics
import subprocess
import sys

import torch
from transformers import Wav2Vec2Config
from transformers import Wav2Vec2ForCTC as HFWav2Vec2ForCTC

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.inference.tts.base_tts_infer import Wav2Vec2ForCTC  # noqa: E402


def flops(cfg, S):
    """Multiply-adds x 2 per clip: the conv stack, the positional conv, the encoder layers (projections, FFN and the two
    attention products) with the feature projection and lm_head."""
    T = specs.w2v_lengths(cfg, S)
    C, H, I = cfg["conv_dim"][0], cfg["hidden_size"], cfg["intermediate_size"]
    conv = 2.0 * T[0] * C * cfg["conv_kernel"][0]
    conv += sum(2.0 * T[i] * C * C * cfg["conv_kernel"][i] for i in range(1, len(T)))
    F = T[-1]
    pos = 2.0 * F * H * (H // cfg["num_conv_pos_embedding_groups"]) * cfg["num_conv_pos_embeddings"]
    layer = 2.0 * F * (4 * H * H + 2 * H * I) + 4.0 * F * F * H
    rest = layer * cfg["num_hidden_layers"] + 2.0 * F * H * (C + cfg["vocab_size"])
    return conv, pos, rest


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("asr_time.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    cfg = specs.W2V_BASE
    sd = specs.synth_w2v(cfg)
    ours, ref = Wav2Vec2ForCTC(Wav2Vec2Config(**cfg)), HFWav2Vec2ForCTC(Wav2Vec2Config(**cfg))
    ours.load_state_dict(sd, strict=True)
    ref.load_state_dict(sd, strict=True)
    ours, ref = ours.eval().to(dev), ref.eval().to(dev)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {q.stdout.strip()}")
    clips = {sec: specs.synth_w2v_wav(sec * specs.W2V_SR, seed=sec).to(dev) for sec in (3, 10, 20)}
    with torch.no_grad():
        for x in clips.values():             # warm every length in both arms
            for _ in range(3):
                ours(x)
                ref(x)
        torch.cuda.synchronize()
        for sec, x in clips.items():
            t = [[], []]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(a.reps):
                for k, f in enumerate((lambda: ours(x), lambda: ref(x))):     # alternated: same clocks and neighbours
                    e0.record()
                    f()
                    e1.record()
                    torch.cuda.synchronize()
                    t[k].append(e0.elapsed_time(e1))
            base = _lib.launch_count()
            got = ours(x).logits
            launches = _lib.launch_count() - base
            want = ref(x).logits
            err = ((got - want).double().pow(2).mean().sqrt() / want.double().pow(2).mean().sqrt()).item()
            conv, pos, rest = flops(cfg, x.shape[1])
            eng, eag = statistics.median(t[0]), statistics.median(t[1])
            sp = lambda v: f"{min(v):.2f}-{max(v):.2f}"
            print(f"{sec:2d} s ({specs.w2v_lengths(cfg, x.shape[1])[-1]} frames, {(conv + pos + rest) / 1e9:.1f} GFLOP: conv stack "
                  f"{conv / 1e9:.1f}, positional conv {pos / 1e9:.1f}, layers {rest / 1e9:.1f}): engine {eng:7.3f} ms (range {sp(t[0])}, "
                  f"{launches} launches)   eager fp32 {eag:7.3f} ms (range {sp(t[1])})   ({eag / eng:.2f}x)   logits rel-RMSE {err:.2e}")
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
                ours(x)
                torch.cuda.synchronize()
            ks = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            print(f"     engine device time {sum(e.device_time_total for e in ks) / 1e3:.3f} ms in {len(ks)} kernels and memsets "
                  f"(profiled pass; the rest of the {eng:.3f} ms call is host work and launch gaps)")
            by = {}
            for e in ks:
                hit = re.search(r"\w*(kernel|memset)\w*", e.name, re.I)
                nm = hit.group(0) if hit else e.name[:32]
                c, us = by.get(nm, (0, 0.0))
                by[nm] = (c + 1, us + e.device_time_total)
            for nm, (c, us) in sorted(by.items(), key=lambda kv: -kv[1][1]):
                print(f"       {nm:32s} x{c:3d} {us / 1e3:8.3f} ms")


if __name__ == "__main__":
    main()
