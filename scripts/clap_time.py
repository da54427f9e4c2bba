"""Time the text-to-audio tool's conditioning (FrozenCLAPEmbedder.encode, audio-chatgpt.py:163-164) on the device at the
shipped shape with seeded synthetic weights: each of T2A's two calls (N = 3 identical prompts, L = 77) on the engine,
its launches, the same seeded BertModel + Projection in eager fp32 PyTorch on the same GPU (TF32 off; when transformers
is importable) with the rel-RMSE between the two, and the DDIM-100 + CFG 1.5 call of the same request (3 clips), so the
conditioning's share of the tool's GPU time comes from one run.  Medians of --reps CUDA-event timings after warm-up,
with the GPU name and power limit read in the same run; a torch.profiler kernel breakdown of one engine encode.

    python scripts/clap_time.py [--reps 20] [--ddim-reps 3]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.ldm.models.diffusion.ddim import DDIMSampler, LatentDiffusionShim  # noqa: E402
from audiogpt_b200.ldm.modules.diffusionmodules.openaimodel import UNetModel  # noqa: E402
from audiogpt_b200.ldm.modules.encoders.modules import FrozenCLAPEmbedder  # noqa: E402


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


class Projection(nn.Module):
    """CLAP/clap.py:8-20 in eval (dropout off)"""

    def __init__(self, d_in, d_out):
        super().__init__()
        self.linear1 = nn.Linear(d_in, d_out, bias=False)
        self.linear2 = nn.Linear(d_out, d_out, bias=False)
        self.layer_norm = nn.LayerNorm(d_out)

    def forward(self, x):
        e1 = self.linear1(x)
        return self.layer_norm(e1 + self.linear2(F.gelu(e1)))


def eager_encoder(cfg, sd):
    import transformers
    bert = transformers.BertModel(transformers.BertConfig(
        vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"], num_hidden_layers=cfg["num_layers"],
        num_attention_heads=cfg["num_heads"], intermediate_size=cfg["intermediate_size"],
        max_position_embeddings=cfg["max_position_embeddings"], type_vocab_size=cfg["type_vocab_size"],
        layer_norm_eps=cfg["layer_norm_eps"]))
    b, p = "caption_encoder.base.", "caption_encoder.projection."
    bert.load_state_dict({k[len(b):]: v for k, v in sd.items() if k.startswith(b)}, strict=True)
    proj = Projection(cfg["hidden_size"], cfg["d_proj"])
    proj.load_state_dict({k[len(p):]: v for k, v in sd.items() if k.startswith(p)}, strict=True)
    bert, proj = bert.eval().cuda(), proj.eval().cuda()
    return lambda ids: proj(bert(input_ids=ids).last_hidden_state), transformers.__version__, \
        bert.config._attn_implementation


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ddim-reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clap_time.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {q.stdout.strip() or torch.cuda.get_device_name()}")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    cfg = specs.CLAP_BASE
    sd = specs.synth_clap(cfg, 7070)
    m = FrozenCLAPEmbedder.from_config(cfg)
    m.load_state_dict(sd, strict=True)
    m = m.eval().cuda()
    g = torch.Generator().manual_seed(5)
    prompt = [101] + torch.randint(1000, cfg["vocab_size"], (9,), generator=g).tolist() + [102]
    rows = {"uc (3 x [''])": [101, 102], "c (3 x [prompt])": prompt}
    ids = {k: torch.tensor([r + [0] * (77 - len(r))] * 3, device="cuda") for k, r in rows.items()}
    out = {}
    total = 0.0
    for name, x in ids.items():
        n0 = _lib.launch_count()
        out[name] = m.encode_ids(x)
        torch.cuda.synchronize()
        launches = _lib.launch_count() - n0
        ms = median_ms(lambda: m.encode_ids(x), a.reps)
        total += ms
        print(f"engine encode {name:18s} N=3 L=77: {ms:8.3f} ms  ({launches} launches per encode)")

    try:
        enc, ver, attn = eager_encoder(cfg, sd)
    except ImportError:
        enc = None
        print("eager fp32 reference: transformers not importable, skipped")
    eager_total = None
    if enc is not None:
        eager_total = 0.0
        with torch.no_grad():
            for name, x in ids.items():
                ref = enc(x)
                ms = median_ms(lambda: enc(x), a.reps)
                eager_total += ms
                e = ((out[name] - ref).double().pow(2).mean().sqrt() / ref.double().pow(2).mean().sqrt()).item()
                print(f"eager fp32 encode {name:14s} N=3 L=77: {ms:8.3f} ms  (transformers {ver}, attn {attn}, "
                      f"TF32 off; rel-RMSE engine vs eager {e:.2e})")
        print(f"conditioning per request: engine {total:.3f} ms, eager fp32 {eager_total:.3f} ms "
              f"({eager_total / total:.2f}x)")

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        m.encode_ids(ids["c (3 x [prompt])"])
        torch.cuda.synchronize()
    print("engine encode kernels (one call):")
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=8))

    ucfg = specs.UNET_TXT2AUDIO
    u = UNetModel(image_size=32, use_checkpoint=True, **ucfg)
    u.load_state_dict(specs.synth_unet(ucfg, 4040), strict=True)
    smp = DDIMSampler(LatentDiffusionShim(u.eval().cuda()).cuda())
    xT = torch.from_numpy(np.random.RandomState(55).randn(3, 4, 10, 78)).to("cuda", torch.float32)
    c, uc = out["c (3 x [prompt])"], out["uc (3 x [''])"]
    ddim = median_ms(lambda: smp.sample(S=100, batch_size=3, shape=(4, 10, 78), conditioning=c, verbose=False, x_T=xT,
                                        eta=0.0, unconditional_guidance_scale=1.5, unconditional_conditioning=uc),
                     a.ddim_reps, warmup=1)
    print(f"DDIM-100 + CFG 1.5, 3 clips, context from the engine's CLAP: {ddim:.1f} ms")
    print(f"conditioning share of (conditioning + DDIM): engine {100 * total / (total + ddim):.2f} %"
          + ("" if eager_total is None else f", eager fp32 {100 * eager_total / (eager_total + ddim):.2f} %"))


if __name__ == "__main__":
    main()
