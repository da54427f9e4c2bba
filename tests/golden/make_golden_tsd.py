#!/usr/bin/env python
"""Generate the target-sound-detection fixtures (tsd_tr125.npz, tsd_branches.npz) by running the REFERENCE's own
RaDur_fusion (audio_detection/target_sound_detection/src/models.py) on CPU fp32 in eval mode, the way the
TargetSoundDetection tool calls it (audio-chatgpt.py:833-848): ``decision, decision_up, logit = model(inputs, embedding)``.

Run in the build container only (needs the reference tree, which does not travel to the GPU box):

    python tests/golden/make_golden_tsd.py

The reference module imports torchlibrosa, which is not installed: torchlibrosa.stft is make_golden_clap_score's
restatement of torchlibrosa 0.1.0 and torchlibrosa.augmentation an empty shell (the eval forward never uses either).
``forward`` builds ``torch.zeros(1).cuda()`` for its unused third output; Tensor.cuda is the identity while it runs.

- tsd_tr125: time_resolution 125 (the tool's default) with every (att_pool, enhancement) pair, on odd, even, >= 1002
  (the stem's 500-row crop) and short (T' < top) clips and two reference lengths.
- tsd_branches: one config in each of the other pool branches (time_resolution 250, 500 and 100).
Every case has its own weights specs.synth_tsd(cfg, weight_seed, out_shift) and mels specs.synth_tsd_mel(T, seed);
neither is stored, only the seeds, the shift, the reference's state-dict keys and shapes, outputs and intermediates
(the reference embedding, the first decision, the top-k indices and values, the final decision).

Seeded weights put most scores near one value, where the gate ``top_k > tao`` is all-or-nothing.  For the enhancement
cases the outputlayer's class-0 bias is shifted (a uniform shift of every logit difference, which keeps the top-k set)
so that tao falls inside the top-k scores, and the case is kept only when every top-k score is at least TAO_MARGIN
from tao, consecutive sorted scores of the top k + 1 differ by at least GAP_MARGIN (so the indices are unambiguous)
and the k-th and (k + 1)-th by at least BOUNDARY_MARGIN (so the top-k set is), the raw top-k mean clears tao by
TAO_MARGIN (so the second pass is mixed in) and every decision_up value is at least HALF_MARGIN from the 0.5 threshold
the tool binarises with.  The margins are several times the largest error the engine shows on an H100.  Otherwise the next mel seed is tried.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, ROOT, save, specs  # noqa: E402
from make_golden_clap_score import torchlibrosa_shim  # noqa: E402

TAO = 0.6
TAO_MARGIN = 2e-3
GAP_MARGIN = 2e-5
HALF_MARGIN = 1e-3
BOUNDARY_MARGIN = 1e-3
TOP = 10

# (att_pool, enhancement, [(T, Tr), ...]) at time_resolution 125
TR125 = [
    (1, 1, [(501, 501), (432, 240), (1010, 501), (40, 240)]),
    (1, 0, [(501, 240), (1010, 501)]),
    (0, 1, [(432, 501), (40, 240)]),
    (0, 0, [(501, 501), (432, 240)]),
]
# (time_resolution, att_pool, enhancement, T, Tr)
BRANCHES = [(250, 1, 0, 501, 501), (500, 0, 0, 432, 240), (100, 1, 0, 501, 240)]


def import_reference_models():
    def shell(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules.setdefault(name, m)
        return sys.modules[name]

    shell("torchlibrosa")
    sys.modules.setdefault("torchlibrosa.stft", torchlibrosa_shim())
    shell("torchlibrosa.augmentation", SpecAugmentation=lambda **k: torch.nn.Identity())
    sys.path.insert(0, os.path.join(REF, "audio_detection"))
    import target_sound_detection.src.models as models
    return models


def build(models, cfg, seed, shift):
    m = models.RaDur_fusion(dict(att_pool=bool(cfg["att_pool"]), enhancement=bool(cfg["enhancement"]), tao=cfg["tao"], top=cfg["top"]),
                            inputdim=64, outputdim=cfg["outputdim"], time_resolution=cfg["time_resolution"])
    m.load_state_dict(specs.synth_tsd(cfg, seed, shift), strict=True)
    return m.eval()


def run(model, x, ref):
    """model(x, ref) with the embedding fed to the first detection pass, the first decision and its top-k captured."""
    cap = {}
    fus = model.detection.fusion.forward

    def fusion_hook(embedding, mix_embed):
        cap.setdefault("embedding", embedding[:, 0].detach().clone())
        return fus(embedding, mix_embed)

    sel = model.select_topk_embeddings

    def select_hook(scores, embeddings, k):
        cap["scores"] = scores.detach().clone()
        cap["topk_idx"] = scores.sort(descending=True, dim=1)[1][:, :k]
        out = sel(scores, embeddings, k)
        cap["topk_val"] = out[1].detach().clone()
        return out

    model.detection.fusion.forward = fusion_hook
    model.select_topk_embeddings = select_hook
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        with torch.no_grad():
            decision, decision_up, _ = model(x, ref)
    finally:
        torch.Tensor.cuda = cuda
        del model.detection.fusion.forward, model.select_topk_embeddings
    return decision, decision_up, cap


def gate_shift(scores, k):
    """The class-0 bias shift that puts tao between two consecutive top-k scores (the lowest split whose top-k mean
    still clears tao), or None."""
    d = torch.logit(scores.double().sort(descending=True)[0][: k + 1])
    lt = float(np.log(TAO / (1 - TAO)))
    for j in range(k - 1, 0, -1):
        delta = lt - 0.5 * (d[j - 1] + d[j]).item()
        p = torch.sigmoid(d + delta)
        if p[:k].mean() > TAO + TAO_MARGIN:
            return delta
    return None


def accept(cfg, cap, decision_up):
    if float((decision_up[..., 0] - 0.5).abs().min()) < HALF_MARGIN:
        return False
    if not cfg["enhancement"]:
        return True
    k = cap["topk_val"].shape[1]
    s = cap["scores"][0].double().sort(descending=True)[0][: k + 1]
    v = cap["topk_val"][0].double()
    boundary = s[k - 1] - s[k] if len(s) > k else float("inf")
    return bool((v - TAO).abs().min() >= TAO_MARGIN and (s[:-1] - s[1:]).min() >= GAP_MARGIN and boundary >= BOUNDARY_MARGIN
                and (v > TAO).any() and (v < TAO).any() and v.mean() > TAO + TAO_MARGIN)


def make_case(models, cfg, wseed, T, Tr, mseed0):
    for mseed in range(mseed0, mseed0 + 100):
        x, ref = specs.synth_tsd_mel(T, mseed), specs.synth_tsd_mel(Tr, mseed + 5000)
        shift = 0.0
        if cfg["enhancement"]:
            _, _, cap = run(build(models, cfg, wseed, 0.0), x, ref)
            k = cap["topk_val"].shape[1]
            delta = gate_shift(cap["scores"][0], k)
            if delta is None:
                continue
            shift = round(delta, 6)
        model = build(models, cfg, wseed, shift)
        decision, decision_up, cap = run(model, x, ref)
        if accept(cfg, cap, decision_up):
            print(f"  T {T} Tr {Tr}: mel seed {mseed}, shift {shift:+.6f}, T' {decision.shape[1]}"
                  + (f", top-k {cap['topk_val'][0].numpy().round(4).tolist()}" if cfg["enhancement"] else ""))
            out = dict(T=np.array(T), Tr=np.array(Tr), mel_seed=np.array(mseed), ref_seed=np.array(mseed + 5000),
                       out_shift=np.array(shift), decision=decision, decision_up=decision_up, embedding=cap["embedding"])
            if cfg["enhancement"]:
                out.update(decision1=cap["scores"], topk_idx=cap["topk_idx"], topk_val=cap["topk_val"])
            return out, model
        print(f"  T {T} Tr {Tr}: mel seed {mseed} rejected")
    raise RuntimeError("no mel seed met the margins")


def keys_and_shapes(model):
    sd = model.state_dict()
    return dict(ref_keys=np.array(list(sd.keys())), ref_shapes=np.array([",".join(str(v) for v in t.shape) for t in sd.values()]))


def main():
    models = import_reference_models()
    arrs = dict(tao=np.array(TAO), top=np.array(TOP), tao_margin=np.array(TAO_MARGIN), gap_margin=np.array(GAP_MARGIN),
                boundary_margin=np.array(BOUNDARY_MARGIN), half_margin=np.array(HALF_MARGIN))
    cases = []
    for ci, (att, enh, lens) in enumerate(TR125):
        cfg = dict(specs.TSD_DEFAULT, att_pool=att, enhancement=enh, top=TOP, tao=TAO)
        print(f"time_resolution 125, att_pool {att}, enhancement {enh}")
        for li, (T, Tr) in enumerate(lens):
            c, model = make_case(models, cfg, 7100 + ci, T, Tr, 1000 * ci + 100 * li)
            cases.append(dict(c, time_resolution=np.array(125), att_pool=np.array(att), enhancement=np.array(enh),
                              weight_seed=np.array(7100 + ci)))
    arrs.update(keys_and_shapes(model))
    for i, c in enumerate(cases):
        arrs.update({f"c{i}_{k}": v for k, v in c.items()})
    save("tsd_tr125", n_cases=np.array(len(cases)), **arrs)

    arrs = dict(tao=np.array(TAO), top=np.array(TOP), half_margin=np.array(HALF_MARGIN))
    for i, (tr, att, enh, T, Tr) in enumerate(BRANCHES):
        cfg = dict(specs.TSD_DEFAULT, time_resolution=tr, att_pool=att, enhancement=enh, top=TOP, tao=TAO)
        print(f"time_resolution {tr}, att_pool {att}, enhancement {enh}")
        c, _ = make_case(models, cfg, 7200 + i, T, Tr, 5000 + 100 * i)
        arrs.update({f"c{i}_{k}": v for k, v in dict(c, time_resolution=np.array(tr), att_pool=np.array(att),
                                                      enhancement=np.array(enh), weight_seed=np.array(7200 + i)).items()})
    save("tsd_branches", n_cases=np.array(len(BRANCHES)), **arrs)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    torch.set_num_threads(os.cpu_count() or 1)
    main()
