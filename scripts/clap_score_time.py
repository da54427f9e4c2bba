"""Time the text-to-audio tool's candidate scoring (T2A.select_best_audio, audio-chatgpt.py:185-199) at its shape: one
prompt (text_len 100) against 3 candidate clips of 159 744 samples at 16 kHz, with seeded synthetic weights of the
shipped CLAP config (Cnn14 + bert-base).  Reports, from one run on the GPU:
- the drop-in's construction from a checkpoint file: the first one (torch.load + packing) and a cached one;
- the engine's select_best_audio work (get_text_embeddings, then get_audio_embeddings + compute_similarity per clip,
  as the tool calls them; host -> device copies of the clips included), median of --reps CUDA-event timings;
- the same arithmetic in eager fp32 PyTorch on the same GPU (oracle/clap_score_ref.py, TF32 off) and the largest
  score difference between the two;
- achieved TFLOP/s of the engine from the FLOPs the shapes need (counted below), and the GPU's name and power limit.

    python scripts/clap_score_time.py [--reps 10]
"""
import argparse
import os
import random
import subprocess
import sys
import tempfile
import time
from unittest import mock

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import specs  # noqa: E402
from audiogpt_b200.wav_evaluation.models import CLAPWrapper as W  # noqa: E402
from oracle import clap_score_ref as ref  # noqa: E402

SR, N_CLIPS, CLIP_LEN, TEXT_LEN = 16000, 3, 159744, 100


class Tok:
    def encode_plus(self, text, add_special_tokens=True, max_length=100, padding="max_length", return_tensors="pt"):
        ids = [101] + [2000 + 37 * i for i in range(9)] + [102]
        pad = max_length - len(ids)
        return {"input_ids": torch.tensor([ids + [0] * pad]), "token_type_ids": torch.zeros(1, max_length, dtype=torch.long),
                "attention_mask": torch.tensor([[1] * len(ids) + [0] * pad])}


def flops(cfg, n_clips, L):
    """FLOPs (2 per MAC) of one select_best_audio call from the shapes: the resampler's FIR, the conv-STFT, the mel
    projection, the 12 convs, fc1, both projections, BERT on L tokens (projections, attention, FFN)."""
    clip = cfg["duration"] * SR
    T, n, F = clip // cfg["hop_size"] + 1, cfg["window_size"], cfg["mel_bins"]
    k, width, o, _ = specs.sinc_resample_kernel(SR, cfg["sampling_rate"])
    per = 2 * clip * k.shape[1] + 2 * T * n * (n + 2) + 2 * T * (n // 2 + 1) * F
    h, w, cin = T, F, 1
    for i, c in enumerate(specs.CNN14_CHANNELS):
        per += 2 * h * w * 9 * (cin * c + c * c)
        cin = c
        if i < len(specs.CNN14_CHANNELS) - 1:
            h, w = h // 2, w // 2
    E, D = cfg["out_emb"], cfg["d_proj"]
    per += 2 * (cin * E + E * D + D * D)
    b = cfg["bert"]
    H, I = b["hidden_size"], b["intermediate_size"]
    text = b["num_layers"] * 2 * L * (4 * H * H + 2 * H * I + 2 * L * H) + 2 * (H * D + D * D)
    return n_clips * per + text, per


def median_ms(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clap_score_time.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {q.stdout.strip() or torch.cuda.get_device_name()}")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    cfg = specs.CLAP_SCORER
    sd = specs.synth_clap_scorer(cfg, 9090)
    rs = np.random.RandomState(1)
    wavs = [(0.1 * rs.randn(CLIP_LEN)).astype(np.float32) for _ in range(N_CLIPS)]
    with tempfile.TemporaryDirectory() as d:
        ckpt, conf = os.path.join(d, "CLAP_weights_2022.pth"), os.path.join(d, "config.yml")
        torch.save({"model": sd}, ckpt)
        with open(conf, "w") as f:
            f.write("".join(f"{k}: {v!r}\n" for k, v in cfg.items() if k != "bert"))
        import transformers
        with mock.patch("transformers.AutoTokenizer.from_pretrained", lambda name: Tok()), \
                mock.patch("transformers.AutoConfig.from_pretrained", lambda name: transformers.BertConfig()):
            ts = []
            for _ in range(2):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                w = W.CLAPWrapper(ckpt, conf, use_cuda=True)
                torch.cuda.synchronize()
                ts.append(1e3 * (time.perf_counter() - t0))
    print(f"construction from the checkpoint: first {ts[0]:.0f} ms, cached {ts[1]:.2f} ms")

    def engine():
        random.seed(0)
        t = w.get_text_embeddings(["a dog barks"])
        return torch.stack([w.compute_similarity(w.get_audio_embeddings([(torch.FloatTensor(x), SR)], resample=True), t,
                                                 use_logit_scale=False).squeeze() for x in wavs])

    sd_gpu = {k: v.cuda() for k, v in sd.items() if v.is_floating_point()}
    tok = Tok().encode_plus("a dog barks", max_length=TEXT_LEN)
    tok = {k: v.cuda() for k, v in tok.items()}

    def eager():
        rng = random.Random()
        rng.seed(0)
        with torch.no_grad():
            t = ref.text_embeddings(sd_gpu, cfg, tok["input_ids"], tok["token_type_ids"], tok["attention_mask"])
            out = []
            for x in wavs:
                c, _ = ref.prepare_clip(torch.from_numpy(x).cuda(), SR, cfg, rng)
                out.append(ref.similarity(ref.audio_embeddings(sd_gpu, cfg, c[None]), t).squeeze())
            return torch.stack(out)

    s_eng, s_eag = engine(), eager()
    ms_eng = median_ms(engine, a.reps)
    ms_eag = median_ms(eager, a.reps)
    total, per = flops(cfg, N_CLIPS, TEXT_LEN)
    print(f"FLOPs: {total / 1e9:.1f} GFLOP per select_best_audio ({per / 1e9:.2f} per candidate)")
    print(f"engine select_best_audio work, {N_CLIPS} x {CLIP_LEN} samples + 1 prompt: {ms_eng:.2f} ms "
          f"({total / ms_eng / 1e9:.1f} TFLOP/s achieved)")
    print(f"eager fp32 PyTorch (TF32 off), same GPU: {ms_eag:.2f} ms ({ms_eag / ms_eng:.2f}x the engine); "
          f"max |score difference| {(s_eng - s_eag).abs().max().item():.2e}, argmax {int(s_eng.argmax())} vs {int(s_eag.argmax())}")


if __name__ == "__main__":
    main()
