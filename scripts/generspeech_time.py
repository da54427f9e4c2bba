"""Time one TTS_OOD request on the device: B = 1, 64 phonemes, a 320-frame reference mel (5.1 s at 16 kHz / hop 256) ->
GenerSpeech (generspeech.yaml: the FS2_C2 front-end, three style levels, the 8-block post-flow) -> HiFi-GAN V1 at 16 kHz.
Seeded synthetic weights (about 5 frames per phoneme).  Prints the median CUDA-event times of the engine and of eager fp32
PyTorch (the CPU oracle run on the GPU with TF32 off) for the acoustic model and the vocoder, with the GPU name and power
limit read in the same run.

    python scripts/generspeech_time.py [--reps 30]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiogpt_b200 import specs  # noqa: E402
from audiogpt_b200.modules.GenerSpeech.model.generspeech import GenerSpeech  # noqa: E402
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator  # noqa: E402
from audiogpt_b200.utils.hparams import set_hparams_from_dict  # noqa: E402
from oracle import generspeech_ref as gr  # noqa: E402
from oracle import hifigan_ref as hr  # noqa: E402


def timed(fn, reps):
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    a, v = [], []
    for i in range(reps + 3):
        e0.record()
        mel = fn[0]()
        e1.record()
        fn[1](mel)
        e2.record()
        torch.cuda.synchronize()
        if i >= 3:
            a.append(e0.elapsed_time(e1))
            v.append(e1.elapsed_time(e2))
    return statistics.median(a), statistics.median(v)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("generspeech_time.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = specs.GS_C2
    set_hparams_from_dict(specs.generspeech_hparams(cfg))
    sd = specs.synth_generspeech(cfg)
    m = GenerSpeech(specs.TokenDictionary(cfg["n_tokens"]))
    m.load_state_dict(sd, strict=True)
    m = m.eval().cuda()
    h = dict(specs.HIFIGAN_V1, audio_sample_rate=16000)
    sdh = specs.synth_hifigan(h)
    voc = HifiGanGenerator(h)
    voc.load_state_dict(sdh, strict=True)
    voc = voc.eval().cuda()
    inp = specs.synth_generspeech_inputs(cfg, 1, 64, 320, seed=5)
    cu = {k: v.cuda() for k, v in inp.items()}
    tok = cu.pop("txt_tokens")
    with torch.no_grad():
        r = m(tok, **cu, global_steps=300000, infer=True)
    m2p = r["mel2ph"]
    z = torch.randn(1, 80, m2p.shape[1], generator=torch.Generator().manual_seed(3)).cuda() * 0.8
    eng = timed((lambda: m(tok, mel2ph=m2p, z_post=z, **cu, global_steps=300000, infer=True)["mel_out"],
                 lambda mel: voc(mel.transpose(1, 2).contiguous())), a.reps)
    sdc = {k: v.cuda() for k, v in sd.items()}
    sdhc = {k: v.cuda() for k, v in sdh.items()}
    args = [cu[k] if k in cu else tok for k in ("txt_tokens", "ref_mels", "ref_mel2ph", "ref_mel2word", "spk_embed", "emo_embed")]
    torch.set_default_device("cuda")     # the oracle builds its index / position tables with default-device factories
    with torch.no_grad():
        eag = timed((lambda: gr.generspeech_forward(sdc, cfg, *args, z, mel2ph=m2p)[0]["mel_out"],
                     lambda mel: hr.hifigan_forward(sdhc, h, mel.transpose(1, 2).contiguous())), a.reps)
        me = m(tok, mel2ph=m2p, z_post=z, **cu, global_steps=300000, infer=True)["mel_out"]
        mo = gr.generspeech_forward(sdc, cfg, *args, z, mel2ph=m2p)[0]["mel_out"]
    torch.set_default_device("cpu")
    err = ((me - mo).double().pow(2).mean().sqrt() / mo.double().pow(2).mean().sqrt()).item()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {q.stdout.strip()}")
    print(f"B=1, 64 phonemes, {m2p.shape[1]} mel frames, 320 reference frames; engine vs eager mel rel-RMSE {err:.2e}")
    print(f"GenerSpeech  engine {eng[0]:.2f} ms   eager fp32 {eag[0]:.2f} ms   ({eag[0] / eng[0]:.2f}x)")
    print(f"HiFi-GAN     engine {eng[1]:.2f} ms   eager fp32 {eag[1]:.2f} ms   ({eag[1] / eng[1]:.2f}x)")
    tot_e, tot_r = sum(eng), sum(eag)
    print(f"TTS_OOD      engine {tot_e:.2f} ms   eager fp32 {tot_r:.2f} ms   ({tot_r / tot_e:.2f}x)")


if __name__ == "__main__":
    main()
