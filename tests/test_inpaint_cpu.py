"""Make-An-Audio Inpaint UNet without a GPU: the CPU oracle against the reference fixtures
(tests/golden/make_golden_inpaint.py), the state-dict layout and head counts against the reference's, and the
install(inpaint=True) routing."""
import os
import subprocess
import sys

import numpy as np
import torch

from audiogpt_b200 import specs
from conftest import load_golden, rel_rmse
from oracle import inpaint_ref as ir, ldm_ref as lr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL_SEED, FULL_SEED = 5050, 6060
SCHEDULE = dict(linear_start=0.0015, linear_end=0.0205)


def test_oracle_small_forwards_and_ddim10_vs_reference():
    g = load_golden("ldm_inpaint_small")
    x, t = torch.tensor(g["x"]), torch.tensor(g["t"])
    for new_order in (False, True):
        for updown in (False, True):
            cfg = dict(specs.UNET_INPAINT_SMALL, use_new_attention_order=new_order, resblock_updown=updown)
            e = rel_rmse(ir.unet_forward(specs.synth_unet(cfg, SMALL_SEED), cfg, x, t),
                         g[f"eps_order{int(new_order)}_updown{int(updown)}"])
            assert e < 1e-5, (new_order, updown, e)
    cfg = specs.UNET_INPAINT_SMALL
    sd = specs.synth_unet(cfg, SMALL_SEED)
    ac = lr.ldm_schedule(**SCHEDULE)["alphas_cumprod"]
    assert torch.equal(ac, torch.tensor(g["alphas_cumprod"]))
    eps_fn = lambda x_, t_, c: ir.unet_forward(sd, cfg, torch.cat([x_, c], 1), t_)
    out = lr.ddim_sample(eps_fn, ac, 10, torch.tensor(g["x_T"]), torch.tensor(g["c"]))
    assert rel_rmse(out, g["ddim10"]) < 1e-4


def test_oracle_shipped_forward_vs_reference():
    g = load_golden("ldm_inpaint")
    cfg = specs.UNET_INPAINT
    eps = ir.unet_forward(specs.synth_unet(cfg, FULL_SEED), cfg, torch.tensor(g["x"]), torch.tensor([991]))
    assert rel_rmse(eps, g["eps"]) < 1e-5


def test_param_shapes_match_reference():
    g = load_golden("ldm_inpaint")
    shapes = specs.unet_param_shapes(specs.UNET_INPAINT)
    assert list(shapes) == list(g["ref_keys"])
    assert [",".join(str(v) for v in s) for s in shapes.values()] == list(g["ref_shapes"])
    assert sum(int(np.prod(s)) for s in shapes.values()) == 107_344_324
    assert "input_blocks.3.0.in_layers.2.weight" in shapes and "output_blocks.2.2.out_layers.3.weight" in shapes
    assert "input_blocks.1.1.qkv.weight" in shapes and shapes["input_blocks.1.1.qkv.weight"] == (960, 320, 1)


def test_planned_heads_match_reference():
    g = load_golden("ldm_inpaint")
    plan = specs.unet_plan(specs.UNET_INPAINT)
    got = []
    for prefix, blocks in (("input_blocks", plan["input_blocks"]), ("middle_block", [plan["middle_block"]]),
                           ("output_blocks", plan["output_blocks"])):
        for i, layers in enumerate(blocks):
            for j, l in enumerate(layers):
                if l[0] == "attn":
                    name = f"{prefix}.{i}.{j}" if prefix != "middle_block" else f"middle_block.{j}"
                    got.append((name, l[2]))
    assert got == list(zip(g["attn_names"], g["attn_heads"].tolist()))
    assert len(got) == 11
    assert [l[3] for b in plan["input_blocks"] for l in b if l[0] == "attn"] == [40, 40, 80, 80]


def test_install_inpaint_routes_attention_unets(tmp_path):
    """install(inpaint=True): UNetModel(...) with the AttentionBlock configs builds AttentionUNetModel; plain install()
    keeps sending them to the reference class (a stub reference module stands in for the reference's)."""
    pkg = tmp_path / "ldm" / "modules" / "diffusionmodules"
    pkg.mkdir(parents=True)
    for d in (tmp_path / "ldm", tmp_path / "ldm" / "modules", pkg):
        (d / "__init__.py").write_text("")
    (pkg / "openaimodel.py").write_text("class UNetModel:\n    def __init__(self, **kw):\n        self.kw = kw\n")
    small = ("dict(image_size=32, in_channels=9, model_channels=64, out_channels=4, num_res_blocks=1, "
             "attention_resolutions=[1], channel_mult=[1], num_heads=2)")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import audiogpt_b200 as a; a.install(inpaint=%s); "
            "import ldm.modules.diffusionmodules.openaimodel as m; from audiogpt_b200 import specs; "
            "from audiogpt_b200.ldm.modules.diffusionmodules.openaimodel import AttentionUNetModel as A; "
            "import audiogpt_b200.ldm.modules.diffusionmodules.openaimodel as ours; "
            "n = [0]; init = A.__init__; A.__init__ = lambda self, **kw: (n.__setitem__(0, n[0] + 1), init(self, **kw))[1]; "
            "u = m.UNetModel(image_size=32, use_checkpoint=True, **specs.UNET_SMALL); "
            "assert type(u) is ours.UNetModel, type(u); "
            "v = m.UNetModel(**" + small + "); w = m.UNetModel(image_size=32, use_checkpoint=True, **specs.UNET_INPAINT); "
            "q = lambda o: type(o).__module__ + '.' + type(o).__name__; "
            "print(q(v), q(w), n[0], sum(p.numel() for p in getattr(w, 'parameters', list)()))")
    outs = {}
    for inpaint in (True, False):
        r = subprocess.run([sys.executable, "-c", code % (str(tmp_path), ROOT, inpaint)], capture_output=True, text=True,
                           timeout=240)
        assert r.returncode == 0, r.stderr
        outs[inpaint] = r.stdout.split()
    ours = "audiogpt_b200.ldm.modules.diffusionmodules.openaimodel.AttentionUNetModel"
    theirs = "ldm.modules.diffusionmodules.openaimodel.UNetModel"
    assert outs[True] == [ours, ours, "2", "107344324"]          # __init__ ran once per model
    assert outs[False] == [theirs, theirs, "0", "0"]
