"""Drop-in for ``modules.fastspeech.fs2.FastSpeech2`` (the acoustic front-end of the TTS and text-to-singing paths).

Reference: /root/reference/NeuralSeq/modules/fastspeech/fs2.py:22-226 with FastspeechEncoder / FastspeechDecoder /
FFTBlocks / DurationPredictor / LengthRegulator / PitchPredictor / EnergyPredictor (modules/fastspeech/tts_modules.py)
and EncSALayer / MultiheadAttention / TransformerFFNLayer / SinusoidalPositionalEmbedding (modules/commons/
common_layers.py).  Same constructor ``(dictionary, out_dims=None)`` reading the global hparams, same
``forward(txt_tokens, mel2ph=None, ..., f0=None, uv=None, energy=None, skip_decoder=False, ...)`` returning the same dict
keys and shapes, same state-dict keys (the shared token embedding under both names, the ``_float_tensor`` buffers, the
``pos_embed_alpha`` parameters), so ``load_ckpt`` loads a reference checkpoint strictly.  Arithmetic: libagpt_b200.so
(csrc/fs2.cu).  CUDA only, inference only.

Covered: encoder_type / decoder_type 'fft', ffn_act 'gelu', ffn_padding 'SAME', dur_loss 'mse', use_pos_embed with
rel_pos false (fairseq table) or true (espnet RelPositionalEncoding), pitch_type 'frame' (use_uv, pitch_norm standard /
log) or 'ph', use_pitch_embed and use_energy_embed on or off, teacher-forced mel2ph / f0 / uv / energy, skip_decoder.
Everything else raises NotImplementedError.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from ... import _lib, paramtree, specs
from ...utils import hparams as _hp

_PITCH_TYPES = {None: 0, "frame": 1, "ph": 2}
_NORMS = {"standard": 1, "log": 2}


def _unsupported(what):
    raise NotImplementedError(f"audiogpt_b200.FastSpeech2 does not support {what}")


def fs2_config(hp, n_tokens, out_dims, use_midi):
    """The engine configuration (specs.fs2_param_shapes / agpt_fs2_cfg) of the reference's hparams; raises
    NotImplementedError for settings outside the covered set."""
    for key, ok in (("encoder_type", "fft"), ("decoder_type", "fft"), ("ffn_act", "gelu"), ("ffn_padding", "SAME"),
                    ("dur_loss", "mse")):
        if hp.get(key, ok) != ok:
            _unsupported(f"{key}={hp.get(key)!r} (only {ok!r})")
    for key in ("use_bert", "use_spk_id", "use_spk_embed", "pitch_ar"):
        if hp.get(key, False):
            _unsupported(f"{key} (speaker conditioning, BERT encoders and autoregressive pitch are out of scope)")
    pitch_type = hp.get("pitch_type") if hp.get("use_pitch_embed") else None
    if pitch_type not in _PITCH_TYPES:
        _unsupported(f"pitch_type={pitch_type!r} (cwt needs an inverse CWT; only 'frame' and 'ph')")
    if pitch_type is not None and hp.get("pitch_norm") not in _NORMS:
        _unsupported(f"pitch_norm={hp.get('pitch_norm')!r} (only 'standard' and 'log')")
    H = int(hp["hidden_size"])
    ph = int(hp.get("predictor_hidden", -1))
    return dict(hidden_size=H, num_heads=int(hp["num_heads"]), enc_layers=int(hp["enc_layers"]),
                dec_layers=int(hp["dec_layers"]), enc_ffn_kernel=int(hp["enc_ffn_kernel_size"]),
                dec_ffn_kernel=int(hp["dec_ffn_kernel_size"]), n_tokens=int(n_tokens), out_dims=int(out_dims),
                predictor_hidden=ph if ph > 0 else H, dur_predictor_layers=int(hp["dur_predictor_layers"]),
                dur_predictor_kernel=int(hp["dur_predictor_kernel"]), predictor_layers=int(hp["predictor_layers"]),
                predictor_kernel=int(hp["predictor_kernel"]), use_pos_embed=int(bool(hp.get("use_pos_embed"))),
                rel_pos=int(bool(hp.get("rel_pos"))), pitch_type=pitch_type,
                use_energy_embed=int(bool(hp.get("use_energy_embed", False))), use_midi=int(use_midi))


class FastSpeech2(nn.Module):
    _use_midi = False
    _h = _lib.engine_handle

    def __init__(self, dictionary, out_dims=None):
        super().__init__()
        hp = _hp.resolve()
        self.dictionary = dictionary
        self.padding_idx = dictionary.pad()
        if self.padding_idx != 0:
            _unsupported(f"a dictionary whose padding index is {self.padding_idx} (the masks treat token 0 as padding)")
        self.enc_layers = int(hp["enc_layers"])
        self.dec_layers = int(hp["dec_layers"])
        self.hidden_size = int(hp["hidden_size"])
        self.out_dims = int(hp["audio_num_mel_bins"]) if out_dims is None else int(out_dims)
        self.cfg = fs2_config(hp, len(dictionary), self.out_dims, self._use_midi)
        self._shapes = specs.fs2_param_shapes(self.cfg)
        for key, shape in self._shapes.items():
            if key == "encoder.embed_tokens.weight":
                continue
            if key.endswith("_float_tensor"):
                paramtree.add_buffer(self, key, torch.zeros(shape))
            else:
                paramtree.add_param(self, key, torch.zeros(shape))
        # FastspeechEncoder holds the same Embedding object as encoder_embed_tokens (fs2.py:30,36)
        paramtree.add_param(self, "encoder.embed_tokens.weight", paramtree.get_param(self, "encoder_embed_tokens.weight"))
        self._engine = _lib.Engine("agpt_fs2_create")

    @torch.no_grad()
    def forward(self, txt_tokens, mel2ph=None, spk_embed=None, ref_mels=None, f0=None, uv=None, energy=None,
                skip_decoder=False, spk_embed_dur_id=None, spk_embed_f0_id=None, infer=False, **kwargs):
        """txt_tokens [B, T_txt] -> {'dur', ['dur_choice'], 'mel2ph', ['pitch_pred', 'f0_denorm'], ['energy_pred'],
        'decoder_inp', ['mel_out']}   (fs2.py:79-138)"""
        return self.run(txt_tokens, mel2ph, f0, uv, energy, skip_decoder, **kwargs)[0]

    @torch.no_grad()
    def run(self, txt_tokens, mel2ph=None, f0=None, uv=None, energy=None, skip_decoder=False, **kwargs):
        """forward's dict, plus the coarse pitch bins that index pitch_embed ([B, T_mel] for 'frame', [B, T_txt] for
        'ph'; None without a pitch embedding)."""
        if not txt_tokens.is_cuda:
            raise RuntimeError("audiogpt_b200.FastSpeech2 runs on CUDA only (no CPU fallback)")
        hp = _hp.resolve()
        dev = txt_tokens.device
        ws = [paramtree.get_tensor(self, k) for k in self._shapes]
        self._engine.ensure(dev, ws, lambda: (
            (C.byref(_lib.Fs2Cfg(**dict(self.cfg, pitch_type=_PITCH_TYPES[self.cfg["pitch_type"]]))),), ws))
        i32 = dict(device=dev, dtype=torch.int32)
        f32 = dict(device=dev, dtype=torch.float32)
        tok = txt_tokens.to(**i32).contiguous()
        B, Tt = tok.shape
        midi = [None, None, None]
        if self._use_midi:
            midi = [kwargs["pitch_midi"].to(**i32).contiguous(),
                    None if kwargs.get("midi_dur") is None else kwargs["midi_dur"].to(**f32).contiguous(),
                    None if kwargs.get("is_slur") is None else kwargs["is_slur"].to(**i32).contiguous()]
        ptr = lambda t: None if t is None else _lib.fptr(t)   # noqa: E731
        ret = {}
        pitch_type = self.cfg["pitch_type"]
        dur = torch.empty((B, Tt), **f32)
        if mel2ph is None:
            dch = torch.empty((B, Tt), **i32)
            mel_len = (C.c_int * B)()
            self._engine.call("fs2_encode", dev, ptr(tok), B, Tt, *map(ptr, midi), 1, ptr(dur), ptr(dch), mel_len)
            Tm = max(mel_len)
            ret["dur"] = dur[:, :, None]
            ret["dur_choice"] = dch.long()
            m2p_in, m2p_out = None, torch.empty((B, Tm), **i32)
        else:
            self._engine.call("fs2_encode", dev, ptr(tok), B, Tt, *map(ptr, midi), 0, ptr(dur), None, None)
            ret["dur"] = dur
            Tm = mel2ph.shape[1]
            m2p_in, m2p_out = mel2ph.to(**i32).contiguous(), None
        grid = Tt if pitch_type == "ph" else Tm
        pitch_pred = f0d = coarse = energy_pred = mel_out = None
        if pitch_type is not None:
            pitch_pred = torch.empty((B, grid, 2 if pitch_type == "frame" else 1), **f32)
            f0d = torch.empty((B, grid), **f32)
            coarse = torch.empty((B, grid), **i32)
        if self.cfg["use_energy_embed"]:
            energy_pred = torch.empty((B, Tm), **f32)
        decoder_inp = torch.empty((B, Tm, self.hidden_size), **f32)
        if not skip_decoder:
            mel_out = torch.empty((B, Tm, self.out_dims), **f32)
        tf = [None if t is None else t.to(**f32).contiguous() for t in (f0, uv, energy)]
        self._engine.call("fs2_decode", dev, Tm, ptr(m2p_in), ptr(m2p_out), *map(ptr, tf), int(bool(hp.get("use_uv"))),
                          _NORMS.get(hp.get("pitch_norm"), 0), float(hp.get("f0_mean", 0.0)), float(hp.get("f0_std", 1.0)),
                          ptr(pitch_pred), ptr(f0d), ptr(coarse), ptr(energy_pred), ptr(decoder_inp), ptr(mel_out))
        ret["mel2ph"] = mel2ph if mel2ph is not None else m2p_out.long()
        if pitch_type is not None:
            ret["pitch_pred"] = pitch_pred
            ret["f0_denorm"] = f0d
        if energy_pred is not None:
            ret["energy_pred"] = energy_pred
        ret["decoder_inp"] = decoder_inp
        if mel_out is not None:
            ret["mel_out"] = mel_out
        return ret, (None if coarse is None else coarse.long())

    @staticmethod
    def mel_norm(x):
        return (x + 5.5) / (6.3 / 2) - 1

    @staticmethod
    def mel_denorm(x):
        return (x + 1) * (6.3 / 2) - 5.5

    def out2mel(self, out):
        return out
