"""Time BASELINE config C2 end to end on the device: 8 utterances of phoneme tokens -> FastSpeech2 (egs/egs_bases/tts/
fs2.yaml: hidden 256, 4 + 4 FFT layers, pitch 'frame') -> HiFi-GAN V1 22.05 kHz.  Seeded synthetic weights; the
synthetic duration predictor gives about 5 frames per token, so the default 130 tokens make about 670 mel frames per
utterance.  Prints FastSpeech2 ms, vocoder ms and
mel frames / s (CUDA events after warm-up), with the GPU name and power limit read in the same run.

    python scripts/fs2_tts_time.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import specs  # noqa: E402
from audiogpt_b200.modules.fastspeech.fs2 import FastSpeech2  # noqa: E402
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator  # noqa: E402
from audiogpt_b200.utils.hparams import set_hparams_from_dict  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--tokens", type=int, default=130, help="tokens per utterance (about 5 frames each)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fs2_tts_time.py needs a CUDA device")
    cfg = specs.FS2_C2
    set_hparams_from_dict(specs.fs2_hparams(cfg))
    fs2 = FastSpeech2(specs.TokenDictionary(cfg["n_tokens"]))
    fs2.load_state_dict(specs.synth_fs2(cfg), strict=True)
    fs2 = fs2.eval().cuda()
    voc = HifiGanGenerator(specs.HIFIGAN_V1).eval().cuda()
    voc.load_state_dict(specs.synth_hifigan(specs.HIFIGAN_V1), strict=True)
    g = torch.Generator().manual_seed(7)
    tok = torch.randint(1, cfg["n_tokens"], (8, a.tokens), generator=g).cuda()

    def step():
        r = fs2(tok)
        e1.record()
        wav = voc(r["mel_out"].transpose(1, 2))
        return r, wav

    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    t_fs2 = t_voc = 0.0
    for _ in range(a.reps):
        e0.record()
        r, wav = step()
        e2.record()
        torch.cuda.synchronize()
        t_fs2 += e0.elapsed_time(e1)
        t_voc += e1.elapsed_time(e2)
    t_fs2 /= a.reps
    t_voc /= a.reps
    frames = int((r["mel2ph"] > 0).sum())
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {q.stdout.strip() or torch.cuda.get_device_name()}")
    print(f"batch 8, {a.tokens} tokens/utt -> {frames} mel frames ({r['mel2ph'].shape[1]} padded), wav {tuple(wav.shape)}")
    print(f"FastSpeech2 {t_fs2:.2f} ms  HiFi-GAN V1 {t_voc:.2f} ms  total {t_fs2 + t_voc:.2f} ms  "
          f"{frames / ((t_fs2 + t_voc) / 1e3):.0f} mel frames/s  (mean of {a.reps} after 3 warm-up steps)")


if __name__ == "__main__":
    main()
