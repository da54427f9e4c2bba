"""Drop-in for ``modules.GenerSpeech.model.generspeech.GenerSpeech`` (the acoustic model of the out-of-domain TTS tool).

Reference: /root/reference/NeuralSeq/modules/GenerSpeech/model/generspeech.py with prosody_util.py (LocalStyleAdaptor,
VQEmbeddingEMA, ProsodyAligner, ConvBlocks), wavenet.py (WN) and glow_modules.py (Glow, CouplingBlock, InvConvNear,
ActNorm).  Same constructor ``(dictionary, out_dims=None)`` reading the global hparams, same state-dict keys (the shared
token embedding and the WN layers the coupling blocks share under every name, weight norm as ``weight_g`` /
``weight_v``, the VQ and InvConvNear buffers), so a reference checkpoint loads strictly.  Arithmetic: libagpt_b200.so
(csrc/generspeech.cu).  CUDA only, inference only.

Covered: the call GenerSpeechInfer.forward_model makes (infer=True, global_steps > forcing), with predicted or
teacher-forced mel2ph, on the FastSpeech2 settings of generspeech.yaml (fft encoder / decoder, fairseq positions, pitch
'frame' with uv and 'standard' norm, no energy) and its post-flow settings.  Returned keys: mel_out (after the post-flow,
2 floor(T_mel / 2) frames), decoder_inp, mel2ph, dur (+ dur_choice when predicted), pitch_pred, f0_denorm, f0_denorm_pred,
ref_prosody, spk_embed, emo_embed, x_mask, ref_mel2ph, ref_mel2word.  The training diagnostics (vq_loss_*, ppl_*, gloss_*,
attn_*) are not computed.  Everything else raises NotImplementedError.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from .... import _lib, paramtree, specs
from ....utils import hparams as _hp
from ...fastspeech.fs2 import fs2_config

_BUFFERS = ("vqvae.data_initialized", "vqvae.embedding", "vqvae.ema_count", "vqvae.ema_weight", "_float_tensor", ".p", ".sign_s",
            ".l_mask", ".eye")


def _unsupported(what):
    raise NotImplementedError(f"audiogpt_b200.GenerSpeech does not support {what}")


def gs_config(hp, n_tokens, out_dims):
    """The engine configuration (specs.generspeech_param_shapes / agpt_gs_cfg) of the reference's hparams; raises
    NotImplementedError outside the covered set."""
    if not hp.get("use_spk_embed", False) or hp.get("use_spk_id", False):
        _unsupported("speaker conditioning other than use_spk_embed (a 256-d speaker embedding)")
    for key, ok in (("post_share_cond_layers", False), ("sigmoid_scale", False), ("use_txt_cond", True)):
        if bool(hp.get(key, ok)) != ok:
            _unsupported(f"{key}={hp.get(key)!r} (only {ok!r})")
    if hp.get("ffn_padding", "SAME") != "SAME":
        _unsupported(f"ffn_padding={hp.get('ffn_padding')!r} (only 'SAME')")
    if int(out_dims) != 80:
        _unsupported(f"out_dims={out_dims} (the post-flow is built for 80 mel bins)")
    cfg = fs2_config(dict(hp, use_spk_embed=False), n_tokens, out_dims, False)
    if cfg["pitch_type"] != "frame" or not hp.get("use_uv") or hp.get("pitch_norm") != "standard":
        _unsupported("a pitch setting other than pitch_type 'frame' with use_uv and pitch_norm 'standard'")
    if cfg["use_energy_embed"] or cfg["rel_pos"] or not cfg["use_pos_embed"]:
        _unsupported("use_energy_embed, rel_pos or no encoder positions")
    return dict(cfg, n_vq=int(hp["nVQ"]), glow_hidden=int(hp["post_glow_hidden"]), glow_kernel=int(hp["post_glow_kernel_size"]),
                glow_blocks=int(hp["post_glow_n_blocks"]), glow_layers=int(hp["post_glow_n_block_layers"]),
                share_wn_layers=int(hp.get("share_wn_layers", 0)))


def _fold(g, v):
    return g * v / v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (v.dim() - 1)))


class GenerSpeech(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, dictionary, out_dims=None):
        super().__init__()
        hp = _hp.resolve()
        self.dictionary = dictionary
        self.padding_idx = dictionary.pad()
        if self.padding_idx != 0:
            _unsupported(f"a dictionary whose padding index is {self.padding_idx} (the masks treat token 0 as padding)")
        self.hidden_size = int(hp["hidden_size"])
        self.out_dims = int(hp["audio_num_mel_bins"]) if out_dims is None else int(out_dims)
        self.cfg = gs_config(hp, len(dictionary), self.out_dims)
        self._shapes = specs.generspeech_param_shapes(self.cfg)
        shared = {"encoder.embed_tokens.weight": "encoder_embed_tokens.weight"}
        for b in range(self.cfg["glow_blocks"]):
            own = specs.gs_wn_owner(self.cfg, b)
            if own != b:
                p, q = f"post_flow.flows.{3 * b + 2}.wn.", f"post_flow.flows.{3 * own + 2}.wn."
                for key in self._shapes:
                    if key.startswith(p) and not key.startswith(p + "cond_layer"):
                        shared[key] = q + key[len(p):]
        for key, shape in self._shapes.items():
            if key in shared:
                continue
            if key.endswith(_BUFFERS):
                paramtree.add_buffer(self, key, torch.zeros(shape))
            else:
                paramtree.add_param(self, key, torch.zeros(shape))
        for key, src in shared.items():
            paramtree.add_param(self, key, paramtree.get_param(self, src))
        self._engine = _lib.Engine("agpt_gs_create")

    def engine_weights(self):
        """The agpt_gs_create weight list: the FastSpeech2 keys, the projections, per prosody level the WN (weight norm
        folded), ConvBlocks, codebook, l1 and aligner, the pitch inpainter, then the post-flow: the blocks' cond_layers
        as one [blocks * 2 hid * layers][2 G] weight, and per block start / end, InvConvNear's inverse (fp32
        torch.inverse of _get_weight(), as the reference's reverse pass computes it), ActNorm bias / logs, and the WN
        layers of the blocks that own them."""
        t = lambda k: paramtree.get_tensor(self, k).detach().float().cpu()   # noqa: E731
        wn = lambda p: _fold(t(p + ".weight_g"), t(p + ".weight_v"))       # noqa: E731
        cfg = self.cfg
        out = [t(k) for k in specs.fs2_param_shapes(cfg)]
        out += [t("spk_embed_proj.weight"), t("spk_embed_proj.bias"), t("emo_embed_proj.weight"), t("emo_embed_proj.bias")]
        for lvl in specs.GS_LEVELS:
            p = f"prosody_extractor_{lvl}"
            for i in range(4):
                out += [wn(f"{p}.wavenet.in_layers.{i}"), t(f"{p}.wavenet.in_layers.{i}.bias")]
            for i in range(4):
                out += [wn(f"{p}.wavenet.res_skip_layers.{i}"), t(f"{p}.wavenet.res_skip_layers.{i}.bias")]
            for r in range(5):
                for j in range(2):
                    q = f"{p}.encoder.res_blocks.{r}.blocks.{j}"
                    out += [t(q + ".0.weight"), t(q + ".0.bias"), t(q + ".1.weight"), t(q + ".1.bias"), t(q + ".4.weight"),
                            t(q + ".4.bias")]
            out += [t(f"{p}.encoder.last_norm.weight"), t(f"{p}.encoder.last_norm.bias"), t(f"{p}.encoder.post_net1.weight"),
                    t(f"{p}.encoder.post_net1.bias"), t(f"{p}.vqvae.embedding"), t(f"l1_{lvl}.weight"), t(f"l1_{lvl}.bias")]
            for i in range(2):
                q = f"align_{lvl}.layers.{i}"
                out += [t(f"{q}.multihead_attn.{n}") for n in ("in_proj_weight", "in_proj_bias", "out_proj.weight", "out_proj.bias")]
                out += [t(f"{q}.{n}") for n in ("linear1.weight", "linear1.bias", "norm1.weight", "norm1.bias", "linear2.weight",
                                                  "linear2.bias", "norm2.weight", "norm2.bias")]
        out += [t(k) for k in self._shapes if k.startswith("pitch_inpainter_predictor.")]
        nb = cfg["glow_blocks"]
        out += [torch.cat([wn(f"post_flow.flows.{3 * b + 2}.wn.cond_layer") for b in range(nb)]),
                torch.cat([t(f"post_flow.flows.{3 * b + 2}.wn.cond_layer.bias") for b in range(nb)])]
        for b in range(nb):
            p = f"post_flow.flows.{3 * b + 2}"
            q = f"post_flow.flows.{3 * b + 1}"
            lw = t(q + ".l") * t(q + ".l_mask") + t(q + ".eye")
            uw = t(q + ".u") * t(q + ".l_mask").transpose(0, 1).contiguous() + torch.diag(t(q + ".sign_s") * torch.exp(t(q + ".log_s")))
            winv = torch.inverse(torch.matmul(t(q + ".p"), torch.matmul(lw, uw)).float())
            out += [wn(p + ".start"), t(p + ".start.bias"), t(p + ".end.weight"), t(p + ".end.bias"), winv,
                    t(f"post_flow.flows.{3 * b}.bias"), t(f"post_flow.flows.{3 * b}.logs")]
            if specs.gs_wn_owner(cfg, b) == b:
                L = cfg["glow_layers"]
                out += [x for i in range(L) for x in (wn(f"{p}.wn.in_layers.{i}"), t(f"{p}.wn.in_layers.{i}.bias"))]
                out += [x for i in range(L) for x in (wn(f"{p}.wn.res_skip_layers.{i}"), t(f"{p}.wn.res_skip_layers.{i}.bias"))]
        return out

    def _engine_cfg(self):
        fs2 = _lib.Fs2Cfg(**{k: (1 if k == "pitch_type" else v) for k, v in self.cfg.items() if k in dict(_lib.Fs2Cfg._fields_)})
        extra = {k: self.cfg[k] for k in ("n_vq", "glow_hidden", "glow_kernel", "glow_blocks", "glow_layers", "share_wn_layers")}
        return _lib.GsConfig(fs2=fs2, **extra)

    def draw_noise(self, shape, device):
        """The post-flow's input noise as run_post_glow draws it: dist.Normal(0, 1).sample(shape) on the CPU generator,
        moved to the device, times hparams['noise_scale']."""
        hp = _hp.resolve()
        return torch.distributions.Normal(0, 1).sample(shape).to(device) * float(hp["noise_scale"])

    @torch.no_grad()
    def forward(self, txt_tokens, mel2ph=None, ref_mel2ph=None, ref_mel2word=None, spk_embed=None, emo_embed=None, ref_mels=None,
                f0=None, uv=None, skip_decoder=False, global_steps=0, infer=False, **kwargs):
        """txt_tokens [B, T_txt], ref_mels [B, T_ref, 80], ref_mel2ph / ref_mel2word [B, T_ref], spk_embed / emo_embed
        [B, 256] -> the dict of GenerSpeech.forward's inference path (see the module docstring).  ``z_post`` in kwargs:
        the post-flow noise [B, 80, T_mel] to use instead of drawing it; ``taps``: a dict to receive the stage outputs
        (mel_pre_flow, prosody_{utter,ph,word}, vq_idx_{utter,ph,word})."""
        hp = _hp.resolve()
        if not infer:
            _unsupported("infer=False (the post-flow's training direction)")
        if global_steps < hp["forcing"]:
            _unsupported(f"global_steps={global_steps} < forcing (the aligners' forced-alignment branch)")
        if f0 is not None or uv is not None or skip_decoder:
            _unsupported("teacher-forced f0 / uv or skip_decoder")
        for name, v in (("ref_mels", ref_mels), ("ref_mel2ph", ref_mel2ph), ("ref_mel2word", ref_mel2word), ("spk_embed", spk_embed),
                        ("emo_embed", emo_embed)):
            if v is None:
                raise ValueError(f"audiogpt_b200.GenerSpeech needs {name}")
        if not txt_tokens.is_cuda:
            raise RuntimeError("audiogpt_b200.GenerSpeech runs on CUDA only (no CPU fallback)")
        dev = txt_tokens.device
        B, Tt = txt_tokens.shape
        if ref_mels.dim() != 3 or ref_mels.shape[0] != B or ref_mels.shape[2] != 80 or ref_mel2ph.shape != ref_mels.shape[:2] or \
                ref_mel2word.shape != ref_mels.shape[:2] or spk_embed.shape != (B, 256) or emo_embed.shape != (B, 256):
            raise ValueError("audiogpt_b200.GenerSpeech: ref_mels [B, T_ref, 80], ref_mel2ph / ref_mel2word [B, T_ref], "
                             "spk_embed / emo_embed [B, 256] expected")
        for name, v in (("ref_mels", ref_mels), ("ref_mel2ph", ref_mel2ph), ("ref_mel2word", ref_mel2word), ("spk_embed", spk_embed),
                        ("emo_embed", emo_embed)):
            if v.device != dev:
                raise RuntimeError(f"audiogpt_b200.GenerSpeech: {name} is on {v.device}, txt_tokens on {dev}")
        ws = [paramtree.get_tensor(self, k) for k in self._shapes]
        self._engine.ensure(dev, ws, lambda: ((C.byref(self._engine_cfg()),), self.engine_weights()))
        i32 = dict(device=dev, dtype=torch.int32)
        f32 = dict(device=dev, dtype=torch.float32)
        ptr = lambda t: None if t is None else _lib.fptr(t)   # noqa: E731
        tok = txt_tokens.to(**i32).contiguous()
        spk_in, emo_in = spk_embed.to(**f32).contiguous(), emo_embed.to(**f32).contiguous()
        H = self.hidden_size
        ret = {}
        dur = torch.empty((B, Tt), **f32)
        spk, emo = torch.empty((B, 1, H), **f32), torch.empty((B, 1, H), **f32)
        if mel2ph is None:
            dch = torch.empty((B, Tt), **i32)
            mel_len = (C.c_int * B)()
            self._engine.call("gs_encode", dev, ptr(tok), B, Tt, ptr(spk_in), ptr(emo_in), 1, ptr(dur), ptr(dch), mel_len,
                              ptr(spk), ptr(emo))
            Tm = max(mel_len)
            ret["dur"], ret["dur_choice"] = dur[:, :, None], dch.long()
            m2p_in, m2p_out = None, torch.empty((B, Tm), **i32)
        else:
            self._engine.call("gs_encode", dev, ptr(tok), B, Tt, ptr(spk_in), ptr(emo_in), 0, ptr(dur), None, None, ptr(spk),
                              ptr(emo))
            ret["dur"] = dur
            Tm = mel2ph.shape[1]
            m2p_in, m2p_out = mel2ph.to(**i32).contiguous(), None
        if Tm < 2:
            raise ValueError(f"audiogpt_b200.GenerSpeech: {Tm} mel frames (the post-flow needs at least 2)")
        z = kwargs.get("z_post")
        if z is None:
            z = self.draw_noise((B, self.out_dims, Tm), dev)
        if tuple(z.shape) != (B, self.out_dims, Tm):
            raise ValueError(f"z_post must be [B, {self.out_dims}, {Tm}]")
        z = z.to(**f32).contiguous()
        refm = ref_mels.to(**f32).contiguous()
        seg_ph, seg_w = ref_mel2ph.to(**i32).contiguous(), ref_mel2word.to(**i32).contiguous()
        n_ph, n_w = int(seg_ph.max()), int(seg_w.max())      # group_hidden_by_segs' torch.max(mel2ph) (a host sync there too)
        if n_ph < 1 or n_w < 1 or int(seg_ph.min()) < 0 or int(seg_w.min()) < 0:
            raise ValueError("audiogpt_b200.GenerSpeech: ref_mel2ph / ref_mel2word must be non-negative with a segment")
        Tr = refm.shape[1]
        pitch_pred = torch.empty((B, Tm, 2), **f32)
        f0d, f0dp = torch.empty((B, Tm), **f32), torch.empty((B, Tm), **f32)
        coarse = torch.empty((B, Tm), **i32)
        decoder_inp, ref_prosody = torch.empty((B, Tm, H), **f32), torch.empty((B, Tm, H), **f32)
        mel_out = torch.empty((B, 2 * (Tm // 2), self.out_dims), **f32)
        taps, taps_c = kwargs.get("taps"), None
        if taps is not None:
            taps["mel_pre_flow"] = torch.empty((B, Tm, self.out_dims), **f32)
            for lvl, n in zip(specs.GS_LEVELS, (Tr, n_ph, n_w)):
                taps["prosody_" + lvl] = torch.empty((B, n, H), **f32)
                taps["vq_idx_" + lvl] = torch.empty((B, n), **i32)
            taps_c = _lib.GsTaps(ptr(taps["mel_pre_flow"]), (C.c_void_p * 3)(*[taps["prosody_" + v].data_ptr() for v in specs.GS_LEVELS]),
                                 (C.c_void_p * 3)(*[taps["vq_idx_" + v].data_ptr() for v in specs.GS_LEVELS]))
        self._engine.call("gs_forward", dev, Tm, ptr(m2p_in), ptr(m2p_out), ptr(refm), Tr, ptr(seg_ph), n_ph, ptr(seg_w), n_w, ptr(z),
                          float(hp.get("f0_mean", 0.0)), float(hp.get("f0_std", 1.0)), ptr(pitch_pred), ptr(f0d), ptr(f0dp), ptr(coarse),
                          ptr(decoder_inp), ptr(ref_prosody), ptr(mel_out), None if taps_c is None else C.byref(taps_c))
        if taps is not None:
            taps["pitch_coarse"] = coarse.long()
        mel2ph = mel2ph if mel2ph is not None else m2p_out.long()
        ret.update(mel2ph=mel2ph, ref_mel2ph=ref_mel2ph, ref_mel2word=ref_mel2word, pitch_pred=pitch_pred, f0_denorm=f0d,
                   f0_denorm_pred=f0dp, decoder_inp=decoder_inp, mel_out=mel_out, x_mask=(mel2ph > 0).float()[:, :, None],
                   spk_embed=spk, emo_embed=emo, ref_prosody=ref_prosody)
        return ret

    @staticmethod
    def mel_norm(x):
        return (x + 5.5) / (6.3 / 2) - 1

    @staticmethod
    def mel_denorm(x):
        return (x + 1) * (6.3 / 2) - 5.5

    def out2mel(self, out):
        return out
