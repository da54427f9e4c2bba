"""Time one SoundExtraction request on the device: a 10 s 32 kHz clip (320 000 samples: T = 626 frames, F = 513 bins)
and an 11-token query -> STFT.transform -> bert-mini + Linear -> UNetRes_FiLM mask -> mask * magnitude ->
STFT.inverse.  Seeded synthetic weights (specs.synth_lass(LASS)).  Prints the median CUDA-event times per stage of the
engine and of eager fp32 PyTorch (oracle/lass_ref.py run on the GPU with TF32 off), the FLOPs counted from the shapes,
and the GPU name and power limit read in the same run.

    python scripts/lass_time.py [--reps 20]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.sound_extraction.model.LASSNet import LASSNet  # noqa: E402
from audiogpt_b200.sound_extraction.utils.stft import STFT  # noqa: E402
from oracle import lass_ref as ref  # noqa: E402

STAGES = ("STFT", "text", "mask", "inverse STFT")


def unet_flops(T, F):
    """Multiply-adds x 2 of UNetRes_FiLM's convs at [1, 1, T, F] (the padded T, the cropped F), FiLM MLPs included."""
    Tp, W = -(-T // 64) * 64, F - 2
    fl, h, w = 0.0, Tp, W
    hs, ws = [], []

    def block(ci, co, h, w):
        f = 2.0 * h * w * 9 * (ci * co + co * co) + (2.0 * h * w * ci * co if ci != co else 0.0)
        return f + 2.0 * (3 if ci != co else 2) * (256 * 2 * co + 2 * co * co)

    for ci, co in specs.LASS_ENC:
        fl += block(ci, co, h, w) + block(co, co, h, w)
        hs.append(h); ws.append(w)
        h, w = h // 2, w // 2
    fl += block(384, 384, h, w)
    for j, (ci, co) in enumerate(specs.LASS_DEC):
        fl += 2.0 * h * w * ci * co * 9                       # ConvTranspose2d: every input pixel x 9 taps
        h, w = hs[-1 - j], ws[-1 - j]
        fl += block(2 * co, co, h, w) + block(co, co, h, w)
    fl += block(32, 32, h, w) + 2.0 * h * w * 32
    return fl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lass_time.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    cfg = specs.LASS
    sd = specs.synth_lass(cfg)
    m = LASSNet.from_config(cfg)
    m.load_state_dict(sd, strict=True)
    m = m.eval().to(dev)
    stft = STFT().to(dev)
    wav = specs.synth_lass_wav(320000, 7)[None].to(dev)
    ids, msk = (t.to(dev) for t in specs.synth_lass_ids(cfg, [11], 8))
    sdc = {k: v.to(dev) for k, v in sd.items()}
    fb, ib = stft.forward_basis, stft.inverse_basis

    def engine():
        mag, phase = yield stft.transform(wav)
        x = mag.transpose(2, 1).unsqueeze(0)
        ids32, m32 = ids.to(torch.int32), msk.to(torch.int32)
        cond = torch.empty(1, 256, device=dev)
        m._ensure(dev)
        yield m._engine.call("lass_text", dev, _lib.fptr(ids32), _lib.fptr(m32), 1, ids.shape[1], _lib.fptr(cond))
        mask = torch.empty_like(x)
        yield m._engine.call("lass_mask", dev, _lib.fptr(x), 1, x.shape[2], x.shape[3], x.stride(0), x.stride(2), x.stride(3),
                             _lib.fptr(cond), _lib.fptr(mask), None)
        yield stft.inverse((mask * x).squeeze(1).permute(0, 2, 1), phase)

    def eager():
        mag, phase = yield ref.stft_transform(wav, fb, specs.LASS_HOP)
        x = mag.transpose(2, 1).unsqueeze(0)
        cond = yield ref.text_cond(sdc, cfg, ids, msk)
        mask = yield torch.sigmoid(ref.unet_logits(sdc, x, cond))
        yield ref.stft_inverse((mask * x).squeeze(1).permute(0, 2, 1), phase, ib, specs.LASS_HOP)

    def timed(gen_fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]
        per = [[] for _ in STAGES]
        tot = []
        for i in range(a.reps + 3):
            g = gen_fn()
            ev[0].record()
            v = next(g)
            for s in range(len(STAGES)):
                ev[s + 1].record()
                try:
                    v = g.send(v)
                except StopIteration:
                    pass
            torch.cuda.synchronize()
            if i >= 3:
                for s in range(len(STAGES)):
                    per[s].append(ev[s].elapsed_time(ev[s + 1]))
                tot.append(ev[0].elapsed_time(ev[-1]))
        return [statistics.median(p) for p in per], statistics.median(tot)

    with torch.no_grad():
        eng, eng_tot = timed(engine)
        eag, eag_tot = timed(eager)
        me = m.forward_ids(stft.transform(wav)[0].transpose(2, 1).unsqueeze(0), ids, msk)
        mag, _ = ref.stft_transform(wav, fb, specs.LASS_HOP)
        mo, _, _ = ref.lass_forward(sdc, cfg, mag.transpose(2, 1).unsqueeze(0), ids, msk)
    err = ((me - mo).double().pow(2).mean().sqrt() / mo.double().pow(2).mean().sqrt()).item()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    T = 320000 // 512 + 1
    fu = unet_flops(T, 513)
    fs = 2.0 * 1026 * 1024 * (320000 + 1024) / 512            # each STFT direction: 1026 x 1024 MACs per frame
    print(f"gpu: {q.stdout.strip()}")
    print(f"1 x 320000 samples (T = {T}, F = 513), 11-token query; engine vs eager mask rel-RMSE {err:.2e}")
    print(f"FLOPs: UNet {fu / 1e9:.1f} G, each STFT direction {fs / 1e9:.2f} G")
    for s, name in enumerate(STAGES):
        extra = f"   engine {fu / eng[s] / 1e9:.1f} TFLOP/s" if name == "mask" else ""
        print(f"{name:13s} engine {eng[s]:8.2f} ms   eager fp32 {eag[s]:8.2f} ms   ({eag[s] / eng[s]:.2f}x){extra}")
    print(f"{'request':13s} engine {eng_tot:8.2f} ms   eager fp32 {eag_tot:8.2f} ms   ({eag_tot / eng_tot:.2f}x)")


if __name__ == "__main__":
    main()
