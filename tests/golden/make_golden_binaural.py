#!/usr/bin/env python
"""Generate the Binaural fixtures (binaural.npz) by running the REFERENCE's own BinauralNetwork
(mono2binaural/src/models.py, use_cuda=False) on CPU fp32, the way the Binaural tool calls it (audio-chatgpt.py:713-773).

Run in the build container only (needs the reference tree, which does not travel to the GPU box):

    python tests/golden/make_golden_binaural.py

Weights (specs.synth_binaural), views (specs.synth_binaural_view) and mono clips (specs.synth_binaural_mono, int16 PCM /
32768 as a loaded wav) are rebuilt from their seeds; the file keeps the seeds, the reference's state-dict keys and shapes,
its frame fields -- ``geometric_warper._warpfield(view, K)`` and ``neural_warpfield(view, K)``, where size = K makes the
nearest interpolation the identity -- and its outputs.

- forward cases c{i}: T = 400 K, K * 400 > T, K * 400 < T, a view with zero quaternions, the small 2 x 16 warpnet.
- chunk-loop runs r{j}: the tool's loop with a view longer than the clip (its m_a slice) and one shorter than it, at a
  reduced chunk_size, and one run at the defaults (chunk_size 48000, rec_field 800) whose rows are the tool's 48000 /
  120 and 48800 / 122 shapes.  Each run also keeps every chunk's frame fields, packed one row after the other.

The generator asserts that the fixtures exercise the three places where the warp is not a plain shift: samples whose
total warp w > 0 was clipped to 0, samples where the clamp at 0 hit, and samples where the running max moved the position.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, save, specs  # noqa: E402

SHIPPED, SMALL = specs.BINAURAL, specs.BINAURAL_SMALL
# (cfg, T, K, zero quaternion frames)
FORWARD = [(SHIPPED, 3200, 8, ()), (SHIPPED, 2001, 7, ()), (SHIPPED, 2999, 5, ()), (SHIPPED, 1600, 4, (0, 2)),
           (SMALL, 4000, 10, ())]
# (L, Kv, chunk_size, rec_field)
RUNS = [(6403, 20, 1600, 800), (6400, 12, 1600, 800), (96000, 240, 48000, 800)]
WEIGHT_SEED = 4242


def reference_net(cfg):
    sys.path.insert(0, os.path.join(REF, "mono2binaural"))
    from src.models import BinauralNetwork
    net = BinauralNetwork(view_dim=7, warpnet_layers=cfg["layers"], warpnet_channels=cfg["channels"], use_cuda=False)
    sd = specs.synth_binaural(cfg, WEIGHT_SEED)
    net.load_state_dict(sd, strict=True)
    return net.eval()


def ref_fields(net, view):
    """the reference's own frame-rate geometric and neural warpfields, [B, 2, K] each"""
    K = view.shape[-1]
    with torch.no_grad():
        return net.warper.geometric_warper._warpfield(view, K), net.warper.neural_warpfield(view, K)


def warp_stats(field, T):
    """(samples with w > 0 clipped, samples clamped at 0, samples the running max moved) of one row"""
    w = F.interpolate(field, size=T)
    pos = torch.clamp(-F.relu(-w) + torch.arange(T, dtype=torch.float32), min=0, max=T - 1)
    raw = -F.relu(-w) + torch.arange(T, dtype=torch.float32)
    return int((w > 0).sum()), int((raw < 0).sum()), int((torch.cummax(pos, dim=-1)[0] != pos).sum())


def tool_loop(net, mono, view, chunk_size, rec_field):
    """audio-chatgpt.py:729-766 after loading: the trims, the chunks, the kept tails, cat and clamp; also each chunk's
    (mono, view) so its frame fields can be stored"""
    if not view.shape[-1] * 400 == mono.shape[-1]:
        mono = mono[:, :(mono.shape[-1] // 400) * 400]
        if view.shape[1] * 400 > mono.shape[1]:
            m_a = view.shape[1] - mono.shape[-1] // 400
            view = view[:, m_a:m_a + (mono.shape[-1] // 400)]
    chunks = [{"mono": mono[:, max(0, i - rec_field):i + chunk_size], "view": view[:, max(0, i - rec_field) // 400:(i + chunk_size) // 400]}
              for i in range(0, mono.shape[-1], chunk_size)]
    for i, chunk in enumerate(chunks):
        with torch.no_grad():
            m = chunk["mono"].unsqueeze(0)
            v = chunk["view"].unsqueeze(0)
            b = net(m, v).squeeze(0)
            if i > 0:
                b = b[:, -(m.shape[-1] - rec_field):]
            chunk["binaural"] = b
    return torch.clamp(torch.cat([c["binaural"] for c in chunks], dim=-1), min=-1, max=1), chunks


def main():
    torch.manual_seed(0)
    nets = {(c["layers"], c["channels"]): reference_net(c) for c in (SHIPPED, SMALL)}
    out = dict(weight_seed=np.int64(WEIGHT_SEED), n_cases=np.int64(len(FORWARD)), n_runs=np.int64(len(RUNS)))
    for k, v in specs.binaural_param_shapes(SHIPPED).items():
        assert tuple(nets[(4, 64)].state_dict()[k].shape) == v, k
    out["keys"] = np.array(list(nets[(4, 64)].state_dict().keys()))
    out["shapes"] = np.array([",".join(map(str, v.shape)) for v in nets[(4, 64)].state_dict().values()])
    totals = np.zeros(3, dtype=np.int64)
    for i, (cfg, T, K, zeros) in enumerate(FORWARD):
        net = nets[(cfg["layers"], cfg["channels"])]
        view = specs.synth_binaural_view(K, seed=100 + i)
        for z in zeros:
            view[:, 3:7, z] = 0.0
        mono = specs.synth_binaural_mono(T, seed=200 + i).unsqueeze(0)
        geo, neu = ref_fields(net, view)
        with torch.no_grad():
            y = net(mono, view)
        totals += warp_stats(geo + neu, T)
        out.update({f"c{i}_layers": np.int64(cfg["layers"]), f"c{i}_channels": np.int64(cfg["channels"]), f"c{i}_T": np.int64(T),
                    f"c{i}_K": np.int64(K), f"c{i}_view_seed": np.int64(100 + i), f"c{i}_mono_seed": np.int64(200 + i),
                    f"c{i}_zero_frames": np.array(zeros, dtype=np.int64), f"c{i}_geometric": geo, f"c{i}_neural": neu, f"c{i}_out": y})
        print(f"forward c{i}: T={T} K={K} layers={cfg['layers']} C={cfg['channels']}")
    net = nets[(4, 64)]
    for j, (L, Kv, cs, rf) in enumerate(RUNS):
        view = specs.synth_binaural_view(Kv, seed=300 + j)[0]
        mono = specs.synth_binaural_mono(L, seed=400 + j)
        y, chunks = tool_loop(net, mono, view, cs, rf)
        fields = []
        for ch in chunks:
            geo, neu = ref_fields(net, ch["view"].unsqueeze(0))
            fields.append((geo + neu)[0].reshape(-1))
            totals += warp_stats(geo + neu, ch["mono"].shape[-1])
        Lo, rows = specs.binaural_chunks(L, Kv, cs, rf)
        assert Lo == y.shape[-1] and len(rows) == len(chunks), (Lo, y.shape, len(rows), len(chunks))
        for r, ch in zip(rows, chunks):
            assert (r["T"], r["K"]) == (ch["mono"].shape[-1], ch["view"].shape[-1])
        out.update({f"r{j}_L": np.int64(L), f"r{j}_Kv": np.int64(Kv), f"r{j}_chunk_size": np.int64(cs), f"r{j}_rec_field": np.int64(rf),
                    f"r{j}_view_seed": np.int64(300 + j), f"r{j}_mono_seed": np.int64(400 + j), f"r{j}_out": y,
                    f"r{j}_fields": torch.cat(fields)})
        print(f"run r{j}: L={L} Kv={Kv} chunk_size={cs}: rows (T, K) {[(r['T'], r['K']) for r in rows]}")
    print(f"clipped w > 0: {totals[0]}, clamped at 0: {totals[1]}, moved by the running max: {totals[2]}")
    assert totals[0] > 0, "no sample has a positive total warp: raise warp_gain or pick other seeds"
    assert totals[1] > 0 and totals[2] > 0
    out["exercised"] = totals
    save("binaural", **out)


if __name__ == "__main__":
    main()
