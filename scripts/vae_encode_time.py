"""Time the first stage's encoder on the device at the Inpaint tool's shape: AutoencoderKLWithEncoder.encode on a
1x80x848 masked mel (shipped first_stage_config, seeded synthetic weights) for B = 1 and 8, and the encode -> decode
round trip forward(x, sample_posterior=False).  Median of --reps CUDA-event timings after warm-up, with the GPU name
and power limit read in the same run, algorithmic TFLOP/s from the FLOP counts of oracle/vae_ref.py and
oracle/vae_enc_ref.py, and, from a separate profiled encode, the share of the tap-GEMM time that the AttnBlocks take.

    python scripts/vae_encode_time.py [--reps 20]
"""
import argparse
import collections
import ctypes as C
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.ldm.models.autoencoder import AutoencoderKLWithEncoder  # noqa: E402
from oracle.vae_enc_ref import vae_encode_flops  # noqa: E402
from oracle.vae_ref import vae_decode_flops  # noqa: E402


def median_ms(fn, reps, warmup=3):
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


def attention_share(m, x):
    """per-launch tap-GEMM records of one encode: the AttnBlock GEMMs are the 1-tap launches that produce q|k|v
    (Cout = 3 Cin), the scores (Cout = tokens), P V (Cin = tokens) and proj_out (residual epilogue, Cin = Cout)"""
    L = _lib.lib()
    torch.cuda.synchronize()
    _lib.check(L.agpt_profile_enable(1))
    try:
        m.encode(x)
        buf = C.create_string_buffer(1 << 22)
        L.agpt_profile_dump(buf, 1 << 22)
    finally:
        _lib.check(L.agpt_profile_enable(0))
    tot = collections.Counter()
    for line in buf.value.decode().splitlines():
        v, G, Ln, Cin, Cout, nt, span, epi, Wr, ms, fl = line.split()
        Ln, Cin, Cout, nt, epi, ms = int(Ln), int(Cin), int(Cout), int(nt), int(epi), float(ms)
        attn = nt == 1 and (Cout == 3 * Cin or Cout == Ln or Cin == Ln or (epi == 1 and Cin == Cout))
        tot["attn" if attn else "other"] += ms
    return tot["attn"], tot["attn"] + tot["other"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_encode_time.py needs a CUDA device")
    cfg = specs.VAE_TXT2AUDIO
    m = AutoencoderKLWithEncoder(ddconfig={k: v for k, v in cfg.items() if k != "embed_dim"},
                                 lossconfig={"target": "torch.nn.Identity"}, embed_dim=cfg["embed_dim"])
    m.load_state_dict(dict(specs.synth_vae_encoder(cfg), **specs.synth_vae_decoder(cfg)), strict=True)
    m = m.eval().cuda()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {q.stdout.strip() or torch.cuda.get_device_name()}")
    H, W = 80, 848
    f_enc = vae_encode_flops(cfg, H, W)
    f_dec = vae_decode_flops(cfg, H // 8, W // 8)
    print(f"algorithmic work per clip: encode {f_enc / 1e9:.1f} GFLOP, decode {f_dec / 1e9:.1f} GFLOP")
    x8 = specs.synth_masked_mel(8, H, W, 848).cuda()
    for B in (1, 8):
        x = x8[:B].contiguous()
        ms = median_ms(lambda: m.encode(x), a.reps)
        print(f"encode    B={B}: {ms:8.2f} ms  {ms / B:7.2f} ms/clip  {f_enc * B / (ms * 1e-3) / 1e12:6.1f} TFLOP/s")
        ms = median_ms(lambda: m(x, sample_posterior=False), a.reps)
        print(f"enc->dec  B={B}: {ms:8.2f} ms  {ms / B:7.2f} ms/clip  {(f_enc + f_dec) * B / (ms * 1e-3) / 1e12:6.1f} TFLOP/s")
    t_attn, t_all = attention_share(m, x8[:1].contiguous())
    print(f"profiled encode B=1: AttnBlock GEMMs {t_attn:.2f} ms of {t_all:.2f} ms tap-GEMM time "
          f"({100 * t_attn / t_all:.1f} %); median of {a.reps} after 3 warm-up calls above")
    fin = torch.isfinite(m.encode(x8[:1]).parameters).all().item()
    print(f"moments finite: {fin}")


if __name__ == "__main__":
    main()
