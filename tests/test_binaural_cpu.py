"""CPU checks of the Binaural tool's BinauralNetwork (mono2binaural/src/models.py): the oracle against the reference's own
outputs and frame fields (tests/golden/binaural.npz, make_golden_binaural.py), the state-dict layout, the chunk plan
and the nearest-frame twin, install(binaural=True), the drop-in's CPU refusal and the C ABI's declarations."""
import os
import re
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import specs  # noqa: E402
from oracle import binaural_ref as ref  # noqa: E402

G = dict(np.load(os.path.join(ROOT, "tests", "golden", "binaural.npz")))
# the oracle restates the reference's fp32 ops in the same order, except the quaternion rotation (fp64 torch against
# scipy's fp64, which may differ in the last bit before the fp32 rounding) and the convs' summation order
FIELD_TOL = 2e-5   # relative to the field's magnitude (hundreds of samples)
OUT_TOL = 1e-5


def case(i):
    c = {k[len(f"c{i}_"):]: v for k, v in G.items() if k.startswith(f"c{i}_")}
    cfg = dict(layers=int(c["layers"]), channels=int(c["channels"]))
    view = specs.synth_binaural_view(int(c["K"]), int(c["view_seed"]))
    for z in c["zero_frames"]:
        view[:, 3:7, int(z)] = 0.0
    mono = specs.synth_binaural_mono(int(c["T"]), int(c["mono_seed"])).unsqueeze(0)
    return c, cfg, specs.synth_binaural(cfg, int(G["weight_seed"])), mono, view


def run(j):
    r = {k[len(f"r{j}_"):]: v for k, v in G.items() if k.startswith(f"r{j}_")}
    view = specs.synth_binaural_view(int(r["Kv"]), int(r["view_seed"]))[0]
    mono = specs.synth_binaural_mono(int(r["L"]), int(r["mono_seed"]))
    return r, mono, view


@pytest.mark.parametrize("i", range(int(G["n_cases"])))
def test_oracle_matches_reference_forward(i):
    c, cfg, sd, mono, view = case(i)
    with torch.no_grad():
        geo = ref.geometric(view)
        neu = ref.neural(sd, cfg, view)
        out = ref.forward(sd, cfg, mono, view)
    scale = np.abs(c["geometric"]).max()
    assert np.abs(geo.numpy() - c["geometric"]).max() <= FIELD_TOL * scale
    assert np.abs(neu.numpy() - c["neural"]).max() <= FIELD_TOL * scale
    assert out.shape == c["out"].shape
    assert np.abs(out.numpy() - c["out"]).max() <= OUT_TOL
    # fed the reference's own frame field, the oracle's warp is the reference's bit for bit
    y = ref.warp(mono, torch.from_numpy(c["geometric"] + c["neural"]))
    assert torch.equal(y, torch.from_numpy(c["out"]))


@pytest.mark.parametrize("j", range(int(G["n_runs"])))
def test_oracle_matches_reference_tool_loop(j):
    r, mono, view = run(j)
    sd = specs.synth_binaural(specs.BINAURAL, int(G["weight_seed"]))
    y = ref.tool(mono, view, lambda m, v: ref.forward(sd, specs.BINAURAL, m, v), int(r["chunk_size"]), int(r["rec_field"]))
    assert y.shape == r["out"].shape
    assert np.abs(y.numpy() - r["out"]).max() <= OUT_TOL
    # and the stored per-chunk fields, packed in the plan's order, reproduce it exactly
    L_out, plan = specs.binaural_chunks(int(r["L"]), int(r["Kv"]), int(r["chunk_size"]), int(r["rec_field"]))
    f, o = torch.from_numpy(r["fields"]), 0
    parts = []
    for p in plan:
        fld = f[o:o + 2 * p["K"]].reshape(1, 2, p["K"])
        o += 2 * p["K"]
        parts.append(ref.warp(mono[:, p["mono_off"]:p["mono_off"] + p["T"]].unsqueeze(0), fld)[0, :, p["keep"]:])
    assert o == f.numel()
    assert torch.equal(torch.clamp(torch.cat(parts, -1), -1, 1), torch.from_numpy(r["out"]))


def test_fixtures_exercise_every_branch():
    clipped, clamped, moved = (int(v) for v in G["exercised"])
    assert clipped > 0 and clamped > 0 and moved > 0
    assert any(len(G[f"c{i}_zero_frames"]) for i in range(int(G["n_cases"])))


def test_state_dict_layout_matches_reference():
    keys = [str(k) for k in G["keys"]]
    shapes = [tuple(int(v) for v in str(s).split(",")) for s in G["shapes"]]
    assert list(specs.binaural_param_shapes(specs.BINAURAL).items()) == list(zip(keys, shapes))
    from audiogpt_b200.mono2binaural.src.models import BinauralNetwork
    net = BinauralNetwork(view_dim=3, use_cuda=False)          # view_dim is ignored, as in the reference
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == list(zip(keys, shapes))
    net.load_state_dict(specs.synth_binaural(specs.BINAURAL), strict=True)
    assert net.num_trainable_parameters() == sum(int(np.prod(s)) for s in shapes)
    assert net.model_name == "binaural_network"


def test_save_and_load_round_trip(tmp_path):
    from audiogpt_b200.mono2binaural.src.models import BinauralNetwork
    a = BinauralNetwork(warpnet_layers=2, warpnet_channels=16, use_cuda=False)
    a.load_state_dict(specs.synth_binaural(specs.BINAURAL_SMALL, 5), strict=True)
    a.save(str(tmp_path))
    b = BinauralNetwork(warpnet_layers=2, warpnet_channels=16, use_cuda=False)
    b.load(str(tmp_path))
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k])


def _tool_slices(L, Kv, cs, rf):
    """the tool's own slicing, observed through oracle.tool with a recording network"""
    mono = torch.arange(L, dtype=torch.float32)[None]
    view = torch.arange(Kv, dtype=torch.float32)[None].repeat(7, 1)
    seen = []

    def net(m, v):
        if v.shape[-1] == 0:
            raise ValueError("empty view")
        seen.append((int(m[0, 0, 0]), m.shape[-1], int(v[0, 0, 0]), v.shape[-1]))
        return torch.arange(m.shape[-1], dtype=torch.float32)[None, None].repeat(1, 2, 1) + 1e6 * len(seen)

    try:
        y = ref.tool(mono, view, net, cs, rf)
    except ValueError:
        return None
    return seen, y


@pytest.mark.parametrize("L,Kv", [(96000, 240), (96000, 300), (96000, 200), (96123, 240), (96123, 241), (48000, 120), (130000, 330),
                                  (1000, 2), (52000, 150), (400, 1), (7999, 19), (200000, 500), (144000, 360), (144399, 359)])
@pytest.mark.parametrize("cs,rf", [(48000, 800), (1600, 800), (4000, 400)])
def test_chunk_plan_matches_tool_slicing(L, Kv, cs, rf):
    got = _tool_slices(L, Kv, cs, rf)
    L_out, plan = specs.binaural_chunks(L, Kv, cs, rf)
    if got is None:
        assert any(p["K"] == 0 for p in plan)
        return
    seen, y = got
    assert all(p["K"] > 0 for p in plan)
    assert [(p["mono_off"], p["T"], p["view_off"], p["K"]) for p in plan] == seen
    assert L_out == y.shape[-1]
    # every row writes rows' kept tails at out_off: tags 1e6 * chunk + sample index
    for n, p in enumerate(plan):
        seg = y[0, p["out_off"]:p["out_off"] + p["T"] - p["keep"]]
        assert seg.numel() == p["T"] - p["keep"]
    expect = torch.cat([torch.arange(p["keep"], p["T"], dtype=torch.float32) + 1e6 * (n + 1) for n, p in enumerate(plan)])
    assert torch.equal(torch.clamp(expect, -1, 1), y[0])


@pytest.mark.parametrize("K", [1, 2, 3, 5, 7, 120, 122, 1001])
@pytest.mark.parametrize("T", [1, 2, 3, 7, 240, 244, 400, 2001, 48000, 48800, 99999])
def test_nearest_twin_matches_interpolate(K, T):
    x = torch.arange(K, dtype=torch.float32)[None, None]
    want = F.interpolate(x, size=T)[0, 0].long().numpy()
    assert np.array_equal(specs.binaural_nearest(T, K), want)


def test_install_binaural_patches_only_the_reference_src():
    import audiogpt_b200
    from audiogpt_b200.mono2binaural.src.models import BinauralNetwork
    names = ("src", "src.models")
    saved = {k: sys.modules.get(k) for k in names}
    try:
        for k in names:
            sys.modules.pop(k, None)
        patched = audiogpt_b200.install(binaural=True)
        assert "src.models (skipped: not importable)" in patched
        assert "src.models" not in sys.modules
        with pytest.raises(ImportError):
            audiogpt_b200.install(strict=True, binaural=True)
        assert not any(p.startswith("src.models") for p in audiogpt_b200.install())
        pkg = types.ModuleType("src")
        pkg.__path__ = []
        # some other project's src.models: left alone
        other = types.ModuleType("src.models")
        other.BinauralNetwork = type("BinauralNetwork", (), {})
        sys.modules.update({"src": pkg, "src.models": other})
        pkg.models = other
        assert "src.models (skipped: not mono2binaural's)" in audiogpt_b200.install(binaural=True)
        assert other.BinauralNetwork is not BinauralNetwork
        with pytest.raises(ImportError):
            audiogpt_b200.install(strict=True, binaural=True)
        # a stand-in of mono2binaural's module: BinauralNetwork is replaced in place, every other name stays
        mod = types.ModuleType("src.models")

        class Theirs:
            pass

        class Warpnet:
            pass

        mod.BinauralNetwork, mod.Warpnet, mod.GeometricWarper = Theirs, Warpnet, Theirs
        sys.modules["src.models"] = mod
        pkg.models = mod
        assert "src.models" in audiogpt_b200.install(binaural=True)
        from src.models import BinauralNetwork as got
        assert got is BinauralNetwork and mod.Warpnet is Warpnet and mod.GeometricWarper is Theirs
        assert sys.modules["src.models"] is mod
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_drop_in_refuses_cpu_tensors():
    from audiogpt_b200.mono2binaural.src.models import BinauralNetwork
    net = BinauralNetwork(use_cuda=False).eval()
    with pytest.raises(RuntimeError, match="CUDA only"):
        net(torch.zeros(1, 1, 800), torch.zeros(1, 7, 2))
    with pytest.raises(RuntimeError, match="CUDA only"):
        net.binauralize(torch.zeros(1, 800), torch.zeros(7, 2))
    with pytest.raises(RuntimeError, match="inference only"):
        net.train()(torch.zeros(1, 1, 800), torch.zeros(1, 7, 2))


def test_header_declares_binaural_abi():
    with open(os.path.join(ROOT, "include", "agpt_b200.h")) as f:
        h = f.read()
    for sym in ("agpt_binaural_create", "agpt_binaural_forward", "agpt_binaural_frames", "agpt_binaural_warp"):
        assert re.search(r"\bint\s+" + sym + r"\s*\(", h), sym
    for t in ("agpt_binaural_cfg", "agpt_binaural_row"):
        assert re.search(r"typedef struct " + t + r"\b", h), t
    from audiogpt_b200 import _lib
    assert [n for n, _ in _lib.BinauralRow._fields_] == ["mono_off", "T", "view_off", "view_stride", "K", "keep", "out_off", "out_stride"]
