"""Time Make-An-Audio's Inpaint chain (audio-chatgpt.py:498-528) on the device at the shipped shape with seeded synthetic
weights, in its four parts: encode the 1x80x848 masked mel (AutoencoderKLWithEncoder), DDIM-100 of the inpainting UNet
with concat conditioning (AttentionUNetModel, on-device loop), decode the 1x4x10x106 latent, BigVGAN on the 80x848 mel.
Median of --reps CUDA-event timings after warm-up, with the GPU name and power limit read in the same run.

    python scripts/inpaint_time.py [--reps 5]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import specs  # noqa: E402
from audiogpt_b200.ldm.models.autoencoder import AutoencoderKLWithEncoder  # noqa: E402
from audiogpt_b200.ldm.models.diffusion.ddim import DDIMSampler, LatentDiffusionShim  # noqa: E402
from audiogpt_b200.ldm.modules.diffusionmodules.openaimodel import AttentionUNetModel  # noqa: E402
from audiogpt_b200.vocoder.bigvgan.models import BigVGAN  # noqa: E402


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
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inpaint_time.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {q.stdout.strip() or torch.cuda.get_device_name()}")

    vcfg = specs.VAE_TXT2AUDIO
    vae = AutoencoderKLWithEncoder(ddconfig={k: v for k, v in vcfg.items() if k != "embed_dim"},
                                   lossconfig={"target": "torch.nn.Identity"}, embed_dim=vcfg["embed_dim"])
    vae.load_state_dict(dict(specs.synth_vae_encoder(vcfg), **specs.synth_vae_decoder(vcfg)), strict=True)
    vae = vae.eval().cuda()
    ucfg = specs.UNET_INPAINT
    unet = AttentionUNetModel(image_size=32, **ucfg)
    unet.load_state_dict(specs.synth_unet(ucfg, 6060), strict=True)
    unet = unet.eval().cuda()
    smp = DDIMSampler(LatentDiffusionShim(unet, linear_start=0.0015, linear_end=0.0205, conditioning_key="concat").cuda())
    hb = specs.BIGVGAN_BASE
    voc = BigVGAN(hb)
    voc.load_state_dict(specs.synth_bigvgan(hb, 4321), strict=True)
    voc = voc.eval().cuda()

    masked_mel = specs.synth_masked_mel(1, 80, 848, 848).cuda()
    mask = -torch.ones(1, 1, 80, 848, device="cuda")
    mask[:, :, :, 300:420] = 1.0
    x_T = torch.from_numpy(np.random.RandomState(55).randn(1, 4, 10, 106)).to("cuda", torch.float32)
    st = {}

    def encode():
        c = vae.encode(masked_mel).mode()
        st["c"] = torch.cat((c, F.interpolate(mask, size=c.shape[-2:])), dim=1)

    def ddim():
        st["z"], st["inter"] = smp.sample(S=100, conditioning=st["c"], batch_size=1, shape=(4, 10, 106), verbose=False,
                                          x_T=x_T)

    def decode():
        st["mel"] = vae.decode(st["z"])

    def vocode():
        st["wav"] = voc(st["mel"][:, 0].clamp(-1, 1))

    parts = [("encode 1x80x848", encode), ("DDIM-100 (100 UNet forwards)", ddim), ("decode 1x4x10x106", decode),
             ("BigVGAN 80x848", vocode)]
    total = 0.0
    for name, fn in parts:
        ms = median_ms(fn, a.reps)
        total += ms
        print(f"{name:32s} {ms:9.2f} ms")
    print(f"{'chain':32s} {total:9.2f} ms   (median of {a.reps} per part)")
    assert len(st["inter"]["x_inter"]) == 2, "DDIM did not take the on-device loop"
    print(f"outputs finite: {bool(torch.isfinite(st['wav']).all())}, waveform samples {st['wav'].numel()}")


if __name__ == "__main__":
    main()
