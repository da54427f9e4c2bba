#!/usr/bin/env python
"""Generate the AutoencoderKL encoder golden fixtures (vae_enc_*.npz) by running the REFERENCE's own modules on CPU fp32,
with the shims and helpers of make_golden.py.

Run in the build container only (needs /root/reference, which does not travel to the GPU box):

    python tests/golden/make_golden_vae_enc.py

vae_enc_small: VAE_SMALL, B=2; vae_enc_txt2audio: the shipped first_stage_config, B=1.  Both encode a 1x80x848 masked
mel (specs.synth_masked_mel, the Inpaint tool's input shape).  The moments are stored in full.  The txt2audio fixture
also runs the reference AutoencoderKL itself (pytorch_lightning stubbed: its LightningModule is nn.Module) and keeps
its state-dict keys / shapes and a strided view of forward(x, sample_posterior=False).
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, import_ldm, save, specs, stats  # noqa: E402

X_SEED = 848


def _stub_lightning():
    pl = types.ModuleType("pytorch_lightning")
    pl.LightningModule = torch.nn.Module
    sys.modules.setdefault("pytorch_lightning", pl)


def _encoder_moments(cfg, sd, x):
    """the reference Encoder + quant_conv, instantiated directly"""
    from ldm.modules.diffusionmodules.model import Encoder
    enc = Encoder(**{k: v for k, v in cfg.items() if k != "embed_dim"})
    print("vae encoder load:", enc.load_state_dict({k[len("encoder."):]: v for k, v in sd.items()
                                                    if k.startswith("encoder.")}, strict=True))
    qc = torch.nn.Conv2d(2 * cfg["z_channels"], 2 * cfg["embed_dim"], 1)
    qc.load_state_dict({"weight": sd["quant_conv.weight"], "bias": sd["quant_conv.bias"]})
    enc.eval()
    with torch.no_grad():
        return qc(enc(x))


def golden_vae_enc():
    x = specs.synth_masked_mel(2, 80, 848, X_SEED)

    cfg = specs.VAE_SMALL
    ms = _encoder_moments(cfg, specs.synth_vae_encoder(cfg), x)
    print("vae_enc small moments rms", ms.pow(2).mean().sqrt().item(), tuple(ms.shape))
    save("vae_enc_small", x_stats=stats(x), moments=ms)

    cfg = specs.VAE_TXT2AUDIO
    sd = dict(specs.synth_vae_encoder(cfg), **specs.synth_vae_decoder(cfg))
    mf = _encoder_moments(cfg, sd, x[:1])
    print("vae_enc txt2audio moments rms", mf.pow(2).mean().sqrt().item(), tuple(mf.shape))

    _stub_lightning()
    from ldm.models.autoencoder import AutoencoderKL
    ae = AutoencoderKL(ddconfig={k: v for k, v in cfg.items() if k != "embed_dim"},
                       lossconfig={"target": "torch.nn.Identity"}, embed_dim=cfg["embed_dim"])
    ref_sd = ae.state_dict()
    print("AutoencoderKL load:", ae.load_state_dict({k: sd[k] for k in ref_sd}, strict=True))
    ae.eval()
    with torch.no_grad():
        rec, post = ae(x[:1], sample_posterior=False)
    assert torch.equal(post.parameters, mf), "AutoencoderKL.encode != Encoder + quant_conv"
    print("vae txt2audio reconstruction rms", rec.pow(2).mean().sqrt().item(), tuple(rec.shape))
    save("vae_enc_txt2audio", x_stats=stats(x[:1]), moments=mf, rec=rec[:, :, ::2, ::3], rec_stats=stats(rec),
         ref_keys=np.array(list(ref_sd.keys())),
         ref_shapes=np.array([",".join(str(v) for v in t.shape) for t in ref_sd.values()]))


if __name__ == "__main__":
    import_ldm()
    cwd = os.getcwd()
    os.chdir(os.path.join(REF, "text_to_audio", "Make_An_Audio"))
    try:
        golden_vae_enc()
    finally:
        os.chdir(cwd)
