"""Time the emotion encoder of one TTS_OOD request on the device: embed_utterance (partials of 160 frames, seeded
weights from specs.synth_emotion) on a 3, 10 and 20 s reference clip at 16 kHz.  The engine and an eager arm on the
same GPU are alternated in one process after every length has been warmed up; times are medians of CUDA-event
intervals around the whole call from a device-resident wav to the device-resident embedding.  The eager arm is the
oracle's mel in torch fp32 (reflect pad, framing, rfft, |.|^2, mel matrix), cuDNN nn.LSTM in fp32 with TF32 off, and
the same slicing, mean and norm.  Also prints the engine's launches per call, its kernels' device time by kernel in
one torch.profiler pass, the embedding's max abs difference between the arms, and the GPU name and power limit read
in the same run.

    python scripts/emotion_time.py [--reps 30]
"""
import argparse
import os
import re
import statistics
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.data_gen.tts.emotion.model import EmotionEncoder  # noqa: E402


class Eager:
    """The eager arm: torch fp32 mel + cuDNN LSTM + slicing, mean and norm."""

    def __init__(self, sd, dev):
        self.lstm = torch.nn.LSTM(40, 256, 3, batch_first=True).to(dev).eval()
        self.lstm.load_state_dict({k[5:]: v for k, v in sd.items() if k.startswith("lstm.")})
        n = specs.EMO_N_FFT
        self.win = torch.hann_window(n, periodic=True, device=dev)
        self.melW = torch.from_numpy(specs.slaney_mel(specs.EMO_SR, n, specs.EMO_MELS, 0.0, specs.EMO_SR / 2.0)).to(dev)

    @torch.no_grad()
    def __call__(self, wav):
        wav_slices, mel_slices = specs.emo_partials(wav.shape[0])
        padded = specs.emo_padded_length(wav.shape[0], wav_slices)
        x = F.pad(wav, (0, padded - wav.shape[0]))
        n = specs.EMO_N_FFT
        x = F.pad(x[None, None], (n // 2, n // 2), mode=specs.EMO_PAD_MODE)[0, 0]
        frames = x.unfold(0, n, specs.EMO_HOP) * self.win
        mel = torch.fft.rfft(frames, dim=1).abs().pow(2) @ self.melW.T
        step = mel_slices[1].start if len(mel_slices) > 1 else 1
        batch = mel.unfold(0, specs.EMO_PARTIAL_FRAMES, step)[:len(mel_slices)].transpose(1, 2)
        _, (h, _) = self.lstm(batch.contiguous())
        raw = h[-1].mean(0)
        return raw / torch.linalg.vector_norm(raw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("emotion_time.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    sd = specs.synth_emotion(specs.EMO)
    ours = EmotionEncoder(dev, torch.device("cpu"))
    ours.load_state_dict(sd, strict=True)
    ours.eval()
    eager = Eager(sd, dev)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {q.stdout.strip()}")
    clips = {sec: torch.from_numpy(specs.synth_emotion_wav(sec * specs.EMO_SR, seed=sec)).to(dev) for sec in (3, 10, 20)}
    arms = (lambda x: ours.engine_embed(x)[0], eager)
    for x in clips.values():                 # warm every length in both arms
        for _ in range(3):
            for f in arms:
                f(x)
    torch.cuda.synchronize()
    for sec, x in clips.items():
        t = [[], []]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.reps):
            for k, f in enumerate(arms):     # alternated: same clocks and neighbours
                e0.record()
                f(x)
                e1.record()
                torch.cuda.synchronize()
                t[k].append(e0.elapsed_time(e1))
        base = _lib.launch_count()
        got = arms[0](x)
        launches = _lib.launch_count() - base
        err = (got - eager(x)).abs().max().item()
        N = len(specs.emo_partials(x.shape[0])[0])
        eng, eag = statistics.median(t[0]), statistics.median(t[1])
        sp = lambda v: f"{min(v):.3f}-{max(v):.3f}"   # noqa: E731
        print(f"{sec:2d} s ({N} partials): engine {eng:7.3f} ms (range {sp(t[0])}, {launches} launches)   eager fp32 {eag:7.3f} ms "
              f"(range {sp(t[1])})   ({eag / eng:.2f}x)   embedding max abs diff {err:.2e}")
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
            arms[0](x)
            torch.cuda.synchronize()
        ks = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        print(f"     engine device time {sum(e.device_time_total for e in ks) / 1e3:.3f} ms in {len(ks)} kernels, copies and memsets "
              f"(profiled pass)")
        by = {}
        for e in ks:
            hit = re.search(r"\w*(kernel|memset|memcpy)\w*", e.name, re.I)
            nm = hit.group(0) if hit else e.name[:32]
            c, us = by.get(nm, (0, 0.0))
            by[nm] = (c + 1, us + e.device_time_total)
        for nm, (c, us) in sorted(by.items(), key=lambda kv: -kv[1][1]):
            print(f"       {nm:32s} x{c:3d} {us / 1e3:8.3f} ms")


if __name__ == "__main__":
    main()
