"""CPU-only tests: the C-ABI library loads and exports every declared symbol, host-side logic
(state-dict layouts, weight-norm folding, schedules, sharding / LPT) and the world_size-2
gloo path of audiogpt_b200.parallel.  No compute calls into the CUDA library here."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from audiogpt_b200 import parallel, specs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_api():
    """(prototypes, structs, defines) parsed from include/agpt_b200.h: {name: (return type, [parameter types])} with
    comments, parameter names and `const` stripped and arrays written as pointers, {agpt_*_cfg: [(field, [array
    lengths])]}, {macro: int}."""
    hdr = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "agpt_b200.h")).read(), flags=re.S)
    defines = {k: int(v) for k, v in re.findall(r"#define\s+(\w+)\s+(\d+)", hdr)}

    def ctype(decl, named=True):
        t = re.sub(r"\[[^]]*\]", "", decl).replace("const", " ")
        if named:
            t = re.sub(r"\w+\s*$", "", t)
        t = re.sub(r"\s*\*\s*", "*", " ".join(t.split())).strip()
        return t + "*" * ("[" in decl)

    protos = {}
    for ret, name, params in re.findall(r"^([A-Za-z_][\w\s\*]*?)\s*\b(agpt_\w+)\s*\(([^)]*)\)\s*;", hdr, re.M | re.S):
        params = [] if params.strip() == "void" else [ctype(p) for p in params.split(",")]
        protos[name] = (ctype(ret, named=False), params)
    structs = {}
    for body, name in re.findall(r"typedef struct \{(.*?)\}\s*(agpt_\w+_cfg)\s*;", hdr, re.S):
        fields = []
        for decl in filter(str.strip, body.split(";")):
            assert decl.strip().startswith("int "), decl
            for f in decl.strip()[len("int"):].split(","):
                dims = [defines[d] for d in re.findall(r"\[(\w+)\]", f)]
                fields.append((f.split("[")[0].strip(), dims))
        structs[name] = fields
    return protos, structs, defines


def test_library_exports_every_declared_symbol():
    """Every declared entry point is exported, and _lib declares its prototype and mirrors its cfg structs exactly."""
    from audiogpt_b200 import _lib
    from audiogpt_b200.build import build
    lib_path = build()
    protos, structs, defines = _header_api()
    assert len(protos) >= 40 and len(structs) == 6
    L = ctypes.CDLL(lib_path)
    for n in protos:
        assert hasattr(L, n), f"{n} declared in include/agpt_b200.h but not exported"
    # the ctypes mirror of every agpt_*_cfg: field names, order, int type and array lengths
    cfg_cls = {f"agpt_{c[:-3].lower()}_cfg": getattr(_lib, c) for c in dir(_lib) if c.endswith("Cfg")}
    assert set(cfg_cls) == set(structs)
    for name, fields in structs.items():
        got = []
        for fname, ft in cfg_cls[name]._fields_:
            dims = []
            while hasattr(ft, "_length_"):
                dims.append(ft._length_)
                ft = ft._type_
            assert ft is ctypes.c_int, (name, fname)
            got.append((fname, dims))
        assert got == fields, name
    assert {k: getattr(_lib, k) for k in defines if k.startswith("AGPT_MAX_")} == \
        {k: v for k, v in defines.items() if k.startswith("AGPT_MAX_")}
    # the declared prototypes: C type -> ctypes type
    scalar = {"int": ctypes.c_int, "long": ctypes.c_long, "long long": ctypes.c_longlong, "float": ctypes.c_float,
              "double": ctypes.c_double, "agpt_handle": ctypes.c_void_p, "agpt_handle*": ctypes.POINTER(ctypes.c_void_p),
              "float**": ctypes.POINTER(ctypes.POINTER(ctypes.c_float))}
    scalar.update({f"{s}*": ctypes.POINTER(cfg_cls[s]) for s in structs})

    def expect(t):
        if t in scalar:
            return scalar[t]
        assert t.endswith("*") and not t.endswith("**"), f"no ctypes rule for the C type {t!r}"
        return ctypes.c_void_p

    assert set(_lib.PROTOTYPES) == set(protos)
    Lp = _lib.lib()
    for n, (ret, params) in protos.items():
        want_ret = None if ret == "void" else ctypes.c_char_p if ret == "char*" else expect(ret)
        want = (want_ret, [expect(p) for p in params])
        assert _lib.PROTOTYPES[n] == want, n
        assert (getattr(Lp, n).restype, getattr(Lp, n).argtypes) == want, n
    assert Lp.agpt_version() >= 100
    assert isinstance(Lp.agpt_last_error(), bytes)


def test_invalid_handle_is_an_error_not_a_crash():
    from audiogpt_b200 import _lib
    L = _lib.lib()
    rc = L.agpt_diffnet_set_cond(None, None, 1, 1, None)
    assert rc != 0 and b"invalid handle" in L.agpt_last_error()


def test_no_cpu_fallback():
    from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator
    m = HifiGanGenerator(specs.HIFIGAN_SMALL)
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(torch.zeros(1, 80, 4))


def test_product_never_imports_oracle():
    bad = []
    for dp, _, fs in os.walk(os.path.join(ROOT, "audiogpt_b200")):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f), errors="ignore").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", txt, re.M):
                    bad.append(f)
    assert not bad, bad


def test_install_aliases_reference_module_names():
    """Without the reference tree on sys.path, install() registers the drop-ins under the reference's
    module names, so `from modules.hifigan.hifigan import HifiGanGenerator` resolves to ours."""
    code = ("import sys; sys.path.insert(0, %r); import audiogpt_b200 as a; p = a.install(); "
            "from modules.hifigan.hifigan import HifiGanGenerator as H; "
            "from ldm.modules.diffusionmodules.openaimodel import UNetModel as U; "
            "from ldm.models.diffusion.ddim import DDIMSampler as D; "
            "from modules.diff.shallow_diffusion_tts import GaussianDiffusion as G; "
            "from vocoder.bigvgan.models import BigVGAN as V; assert V.__module__.startswith('audiogpt_b200'); "
            "assert H.__module__.startswith('audiogpt_b200') and U.__module__.startswith('audiogpt_b200'); "
            "assert D.__module__.startswith('audiogpt_b200') and G.__module__.startswith('audiogpt_b200'); "
            "print(len(p))") % ROOT
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip() == "8"


def test_install_keeps_reference_unet_for_unsupported_configs(tmp_path):
    """install() replaces UNetModel inside the reference module; AudioGPT also builds UNets outside this back-end's
    scope (the inpainting AttentionBlock UNet: use_spatial_transformer=False).  Those configs must still construct --
    as instances of the reference's own class -- while the txt2audio config gets the drop-in (VERDICT r1 #8)."""
    pkg = tmp_path / "ldm" / "modules" / "diffusionmodules"
    pkg.mkdir(parents=True)
    for d in (tmp_path / "ldm", tmp_path / "ldm" / "modules", pkg):
        (d / "__init__.py").write_text("")
    (pkg / "openaimodel.py").write_text("class UNetModel:\n    def __init__(self, **kw):\n        self.kw = kw\n")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import audiogpt_b200 as a; a.install(); "
            "import ldm.modules.diffusionmodules.openaimodel as m; from audiogpt_b200 import specs; "
            "u = m.UNetModel(image_size=32, use_checkpoint=True, **specs.UNET_SMALL); "
            "assert type(u).__module__.startswith('audiogpt_b200'), type(u); "
            "v = m.UNetModel(image_size=32, in_channels=9, model_channels=64, out_channels=4, num_res_blocks=1, "
            "attention_resolutions=[1], channel_mult=[1], num_heads=2); "
            "assert type(v).__module__ == 'ldm.modules.diffusionmodules.openaimodel' and v.kw['in_channels'] == 9; "
            "print('ok')") % (str(tmp_path), ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr
    # without install() there is no reference class to route to: unsupported configs raise
    from audiogpt_b200.ldm.modules.diffusionmodules.openaimodel import UNetModel
    with pytest.raises(NotImplementedError, match="AttentionBlock"):
        UNetModel(image_size=32, in_channels=9, model_channels=64, out_channels=4, num_res_blocks=1,
                  attention_resolutions=[1], channel_mult=[1], num_heads=2)


def test_param_tables_match_survey_counts():
    n = lambda shapes: sum(int(np.prod(s)) for s in shapes.values())
    assert n(specs.hifigan_param_shapes(specs.HIFIGAN_V1)) == 13_926_017   # 13.93 M (SURVEY 8a)
    assert abs(n(specs.diffnet_param_shapes(specs.DIFFNET_BASE)) / 15.09e6 - 1) < 0.01
    assert abs(n(specs.unet_param_shapes(specs.UNET_TXT2AUDIO)) / 160.2e6 - 1) < 0.01
    plan = specs.unet_plan(specs.UNET_TXT2AUDIO)
    assert len(plan["input_blocks"]) == 6 and len(plan["output_blocks"]) == 6
    kinds = [[l[0] for l in b] for b in plan["output_blocks"]]
    assert kinds[2] == ["res", "st", "up"] and plan["output_blocks"][0][0][1:3] == (1280, 640)
    assert plan["output_blocks"][2][0][1:3] == (960, 640) and plan["output_blocks"][3][0][1:3] == (960, 320)


def test_weight_norm_fold_matches_torch():
    from audiogpt_b200.modules.hifigan.hifigan import fold_weight_norm
    g = torch.Generator().manual_seed(0)
    for shape in [(8, 4, 3), (6, 5, 16)]:      # Conv1d [Cout,Cin,k] and ConvTranspose1d [Cin,Cout,k]
        v = torch.randn(shape, generator=g)
        gg = torch.rand((shape[0], 1, 1), generator=g) + 0.5
        ref = torch._weight_norm(v, gg, 0)
        assert torch.allclose(fold_weight_norm(gg, v), ref, atol=1e-6)


def test_hifigan_state_dict_roundtrip_both_layouts():
    from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator
    h = specs.HIFIGAN_SMALL
    m = HifiGanGenerator(h)
    sd_wn = m.state_dict()
    assert any(k.endswith("weight_g") for k in sd_wn)
    m2 = HifiGanGenerator(h)
    m2.load_state_dict(sd_wn, strict=True)
    m2.remove_weight_norm()
    assert list(m2.state_dict().keys()).count("conv_pre.weight") == 1
    m3 = HifiGanGenerator(h)                       # folded checkpoint into a fresh (weight-normed) module
    m3.load_state_dict(m2.state_dict(), strict=True)
    for a, b in zip(m2.folded_weights(), m3.folded_weights()):
        assert torch.equal(a, b)
    m4 = HifiGanGenerator(h)
    m4.remove_weight_norm()                        # g/v checkpoint into an already-folded module
    m4.load_state_dict(sd_wn, strict=True)
    for a, b in zip(m2.folded_weights(), m4.folded_weights()):
        assert torch.allclose(a, b, atol=1e-7)


def test_gaussian_diffusion_buffers_and_plms_scalars():
    from audiogpt_b200.modules.diff import shallow_diffusion_tts as sdt
    from audiogpt_b200.utils.hparams import set_hparams_from_dict
    from oracle import diffusion_ref as dr
    set_hparams_from_dict(dict(specs.DIFFNET_SMALL, keep_bins=80, schedule_type="linear", max_beta=0.06))
    gd = sdt.GaussianDiffusion(None, 80, torch.nn.Identity(), timesteps=100, K_step=100,
                               spec_min=specs.SPEC_MIN, spec_max=specs.SPEC_MAX)
    tab = dr.schedule_tables(dr.linear_betas(100, 0.06))
    for k, v in tab.items():
        assert torch.equal(getattr(gd, k), v), k
    # fused PLMS scalars reproduce get_x_pred
    x, e = torch.randn(1, 1, 80, 5), torch.randn(1, 1, 80, 5)
    for tv in (99, 50, 7):
        a, b = gd._plms_scalars(tv, 10)
        ref = dr.plms_x_pred(tab, x, e, torch.tensor([tv]), 10)
        assert torch.allclose(a * x + b * e, ref, atol=1e-5)


def test_ddim_tables_match_oracle():
    from audiogpt_b200.ldm.models.diffusion.ddim import DDIMSampler, LatentDiffusionShim
    from oracle import ldm_ref as lr
    ldm = LatentDiffusionShim(torch.nn.Identity())
    s = DDIMSampler(ldm)
    s.make_schedule(100, ddim_eta=0.0, verbose=False)
    tab = lr.ddim_tables(lr.ldm_schedule()["alphas_cumprod"], 100)
    assert np.array_equal(s.ddim_timesteps, tab["timesteps"]) and s.ddim_timesteps[0] == 1 and s.ddim_timesteps[-1] == 991
    assert torch.equal(s.ddim_alphas.cpu(), torch.as_tensor(tab["alphas"]))
    assert np.array_equal(np.asarray(s.ddim_alphas_prev, dtype=np.float64), np.asarray(tab["alphas_prev"], dtype=np.float64))


def test_shard_range_and_lpt():
    assert [parallel.shard_range(32, 8, r) for r in range(8)] == [(4 * r, 4 * r + 4) for r in range(8)]
    assert [parallel.shard_range(10, 4, r) for r in range(4)] == [(0, 3), (3, 6), (6, 9), (9, 10)]
    assert parallel.shard_range(2, 4, 3) == (2, 2)
    rng = np.random.RandomState(7)
    costs = [parallel.job_cost_tflop("tts", int(t)) for t in rng.randint(200, 801, 32)] + \
            [parallel.job_cost_tflop("t2a")] * 32
    asg = parallel.lpt_assign(costs, 8)
    assert sorted(i for w in asg for i in w) == list(range(64))
    loads = [sum(costs[i] for i in w) for w in asg]
    assert max(loads) / (sum(costs) / 8) < 1.05          # 32 equal big jobs over 8 GPUs + small fill
    assert all(sum(1 for i in w if i >= 32) == 4 for w in asg)


WORKER = r"""
import os, sys, torch
sys.path.insert(0, {root!r})
from audiogpt_b200 import parallel, specs
rank, world, local = parallel.init_distributed("gloo")
assert world == 2
h = specs.HIFIGAN_SMALL
shapes = specs.hifigan_param_shapes(h)
sd = specs.synth_hifigan(h, 1234) if rank == 0 else {{k: torch.zeros(s) for k, s in shapes.items()}}
sd = parallel.broadcast_state_dict(sd, src=0)
ref = specs.synth_hifigan(h, 1234)
assert all(torch.equal(sd[k], ref[k]) for k in ref), "broadcast mismatch"
lo, hi = parallel.shard_range(5, world, rank)          # ragged: 3 + 2 utterances
mine = torch.arange(lo, hi, dtype=torch.float32)[:, None, None].expand(hi - lo, 1, 7).contiguous()
allw = parallel.all_gather_rows(mine, counts=[3, 2])
assert allw.shape == (5, 1, 7) and torch.equal(allw[:, 0, 0], torch.arange(5.0))
eq = parallel.all_gather_rows(torch.full((2, 3), float(rank)))
assert eq.shape == (4, 3) and eq[0, 0] == 0 and eq[3, 0] == 1
# mixed dtypes keep their dtype and value (ADVICE r1): an int64 buffer above 2^24 and a half tensor
mixed = {{"w": torch.full((3,), 1.5 if rank == 0 else 0.0), "n": torch.tensor([2 ** 40 + 1 if rank == 0 else 0]),
         "h": torch.full((2,), 0.25 if rank == 0 else 0.0, dtype=torch.float16)}}
got = parallel.broadcast_state_dict(mixed, src=0)
assert got["n"].dtype == torch.int64 and int(got["n"][0]) == 2 ** 40 + 1 and got["h"].dtype == torch.float16
assert float(got["w"][0]) == 1.5 and float(got["h"][1]) == 0.25 and list(got) == ["w", "n", "h"]
# disagreement on the key/shape list is detected on every rank instead of silently mis-slicing the blob
bad = {{"w": torch.zeros(3 + rank)}}
try:
    parallel.broadcast_state_dict(bad, src=0)
    raise SystemExit("shape mismatch not detected")
except RuntimeError as ex:
    assert "disagree" in str(ex)
# asynchronous gather (the bench's waveform all-gather): two batches in flight, drained in order
ag = parallel.AsyncGather()
ag.submit(torch.full((2, 4), 10.0 + rank)); ag.submit(torch.full((1, 4), 20.0 + rank))
g0, g1 = ag.drain()
assert g0.shape == (4, 4) and g0[0, 0] == 10 and g0[3, 0] == 11 and g1.shape == (2, 4) and g1[1, 0] == 21
# mixed dispatch (BASELINE configs[4]): LPT assignment, every job exactly once, one all_gather of timings
import time
jobs = [("tts", 200 + 37 * i) for i in range(6)] + [("t2a", 0)] * 2
done = []
res = parallel.run_mixed(jobs, lambda i, kind, frames: (done.append(i), time.sleep(0.01 if kind == "tts" else 0.05)))
assert sorted(res["assignment"][0] + res["assignment"][1]) == list(range(8))
assert done == res["assignment"][rank] and len(res["busy_s"]) == 2
assert res["makespan_s"] >= max(res["busy_s"]) - 1e-9 and abs(max(res["busy_fraction"]) - 1.0) < 1e-9
assert abs(res["model_load_tflop"][0] - res["model_load_tflop"][1]) < 1.0     # one t2a clip (~19 TFLOP) on each rank
# grouped service: a rank serves its own jobs of one kind in micro-batches (the bench's text-to-audio batches of 4)
groups = []
res2 = parallel.run_mixed([("tts", 300)] * 4 + [("t2a", 0)] * 6, None, run_group=lambda kind, idxs: groups.append((kind, list(idxs))),
                          group_size=dict(t2a=2))
mine = res2["assignment"][rank]
assert sorted(i for _, g in groups for i in g) == sorted(mine)
assert all(len(g) <= (2 if k == "t2a" else 1) for k, g in groups) and sum(len(g) for k, g in groups if k == "t2a") == 3
print("rank", rank, "ok", flush=True)
import torch.distributed as dist
dist.barrier()
dist.destroy_process_group()
os._exit(0)        # skip interpreter teardown (gloo/TCPStore threads racing at exit made this flaky)
"""


def test_world_size_2_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=ROOT))
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE="2", CUDA_VISIBLE_DEVICES="")
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r), LOCAL_RANK=str(r)),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=240)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, o
        assert f"rank {r} ok" in o


def test_bigvgan_state_dict_layouts_and_abi_order():
    """BigVGAN drop-in: strict load of a folded checkpoint, weight-norm round trip, and the weight list handed to
    the C ABI (state-dict order without the Activation1d filter buffers, then the 12 taps once)."""
    from audiogpt_b200.vocoder.bigvgan.models import BigVGAN
    h = specs.BIGVGAN_SMALL
    sd = specs.synth_bigvgan(h, 4321)
    m = BigVGAN(h)
    assert any(k.endswith("weight_g") for k in m.state_dict())
    m.load_state_dict(sd, strict=True)                   # folded checkpoint into a weight-normed module
    assert set(m.state_dict()) == set(sd)
    fw = m.folded_weights()
    n_act = sum(1 for k in sd if k.endswith(".act.alpha"))
    assert n_act == 4 * 3 * 6 + 1 and len(fw) == len(sd) - 2 * n_act + 1
    assert fw[-1].shape == (12,) and abs(float(fw[-1].sum()) - 1.0) < 1e-6
    assert torch.equal(fw[0], sd["conv_pre.weight"]) and torch.equal(fw[-3], sd["conv_post.weight"])
    m2 = BigVGAN(h)                                       # g/v checkpoint -> folded module
    sd_wn = m2.state_dict()
    m3 = BigVGAN(h)
    m3.remove_weight_norm()
    m3.load_state_dict(sd_wn, strict=True)
    for a, b in zip(m2.folded_weights(), m3.folded_weights()):
        assert torch.allclose(a, b, atol=1e-7)
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(torch.zeros(1, 80, 4))


# ---- bench.py contract of the reference arm (CPU only: it is the one arm that must run without a GPU)
def test_bench_reference_arm_contract():
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    env.pop("RANK", None)
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=600, env=env, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip().startswith("{")]
    assert len(lines) == 1                                   # ONE JSON line
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "mel_frames_per_s_vocoded" and d["unit"] == "frames/s"
    assert d["higher_is_better"] is True and d["n_gpus"] == 1 and d["steps"] == 1 and d["value"] > 0
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["value"] == d["value"] and cb["cores"] >= 1 and "mallopt" in cb["sample"]
    assert abs(d["ms_per_step"] * 1e-3 * d["value"] - d["frames_per_step"]) < 1e-3 * d["frames_per_step"]   # nothing extrapolated
    assert d["ddim"]["metric"] == "clips_per_s_ddim100_cfg" and d["ddim"]["value"] > 0
    # every other rank of a torchrun launch exits 0 without work and without output
    env["RANK"] = "1"
    r1 = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                        capture_output=True, text=True, timeout=120, env=env, cwd=root)
    assert r1.returncode == 0 and r1.stdout.strip() == ""


def _header():
    return re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "agpt_b200.h")).read(), flags=re.S)


def _header_struct_fields(name):
    """(field name, ctypes type) of the tagged struct `name` of the header, in declaration order"""
    body = re.search(r"typedef struct %s \{(.*?)\}\s*%s;" % (name, name), _header(), re.S).group(1)
    want = []
    for decl in filter(str.strip, body.split(";")):
        decl = decl.replace("const", " ").strip()
        ptr = "*" in decl
        t = decl.split()[0]
        for field in decl.split(None, 1)[1].replace("*", " ").split(","):
            ct = ctypes.c_void_p if ptr else {"int": ctypes.c_int, "long": ctypes.c_long, "float": ctypes.c_float}[t]
            want.append((field.strip(), ct))
    return want


def test_tapconv_probe_args_mirror_the_header():
    """_lib.TapconvProbeArgs has the fields of agpt_tapconv_probe_args in the header's order and C types (a mismatch
    would hand the probe shifted launch parameters)."""
    from audiogpt_b200 import _lib
    want = _header_struct_fields("agpt_tapconv_probe_args")
    got = [(n, t) for n, t in _lib.TapconvProbeArgs._fields_]
    assert [t for _, t in got] == [t for _, t in want]
    assert [n for n, _ in got] == [("inp" if n == "in" else n) for n, _ in want]   # `in` is a Python keyword


def test_tapconv_pipes_and_kernel_ids_mirror_the_header():
    """_lib.TapconvPipes has the fields of agpt_tapconv_pipes, and _lib.TC_KERNS lists the AGPT_TC_KERN_* kernel
    families of agpt_tapconv_probe_pipes's ran[4] in the enum's order (a mismatch would set the wrong pipeline or let
    a case assert the wrong kernel)."""
    from audiogpt_b200 import _lib
    assert [(n, t) for n, t in _lib.TapconvPipes._fields_] == _header_struct_fields("agpt_tapconv_pipes")
    enum = re.search(r"enum \{([^}]*AGPT_TC_KERN_TILE[^}]*)\}", _header(), re.S).group(1)
    names = [e.split("=")[0].strip() for e in enum.split(",") if e.strip()]
    assert names == ["AGPT_TC_KERN_" + n for n in _lib.TC_KERNS]
    assert "AGPT_TC_KERN_TILE = 0" in enum and enum.count("=") == 1


def test_nn_probe_args_mirror_the_header():
    """_lib.NnProbeArgs has the fields of agpt_nn_probe_args in the header's order and C types, and _lib.NN_OPS lists
    the AGPT_NN_* selectors in the enum's order (a mismatch would run another kernel or shift its arguments)."""
    from audiogpt_b200 import _lib
    want = _header_struct_fields("agpt_nn_probe_args")
    assert [(n, t) for n, t in _lib.NnProbeArgs._fields_] == want
    enum = re.search(r"enum \{([^}]*AGPT_NN_GROUPNORM[^}]*)\}", _header(), re.S).group(1)
    names = [e.split("=")[0].strip() for e in enum.split(",") if e.strip()]
    assert names == ["AGPT_NN_" + n for n in _lib.NN_OPS]
    assert "AGPT_NN_GROUPNORM = 0" in enum and enum.count("=") == 1


def test_fs_probe_args_mirror_the_header():
    """_lib.FsProbeArgs has the fields of agpt_fs_probe_args in the header's order and C types, and _lib.FS_OPS lists
    the AGPT_FS_* selectors in the enum's order (a mismatch would run another kernel or shift its arguments)."""
    from audiogpt_b200 import _lib
    want = _header_struct_fields("agpt_fs_probe_args")
    assert [(n, t) for n, t in _lib.FsProbeArgs._fields_] == want
    enum = re.search(r"enum \{([^}]*AGPT_FS_EMBED_TOKENS[^}]*)\}", _header(), re.S).group(1)
    names = [e.split("=")[0].strip() for e in enum.split(",") if e.strip()]
    assert names == ["AGPT_FS_" + n for n in _lib.FS_OPS]
    assert "AGPT_FS_EMBED_TOKENS = 0" in enum and enum.count("=") == 1


def test_audio_probe_args_mirror_the_header():
    """_lib.AudioProbeArgs has the fields of agpt_audio_probe_args in the header's order and C types, and _lib.AU_OPS
    lists the AGPT_AU_* selectors in the enum's order (a mismatch would run another kernel or shift its arguments)."""
    from audiogpt_b200 import _lib
    want = _header_struct_fields("agpt_audio_probe_args")
    assert [(n, t) for n, t in _lib.AudioProbeArgs._fields_] == want
    enum = re.search(r"enum \{([^}]*AGPT_AU_FRAMES[^}]*)\}", _header(), re.S).group(1)
    names = [e.split("=")[0].strip() for e in enum.split(",") if e.strip()]
    assert names == ["AGPT_AU_" + n for n in _lib.AU_OPS]
    assert "AGPT_AU_FRAMES = 0" in enum and enum.count("=") == 1


def test_voc_probe_args_mirror_the_header():
    """_lib.VocProbeArgs has the fields of agpt_voc_probe_args in the header's order and C types, and _lib.VC_OPS lists
    the AGPT_VC_* selectors in the enum's order (a mismatch would run another kernel or shift its arguments)."""
    from audiogpt_b200 import _lib
    want = _header_struct_fields("agpt_voc_probe_args")
    assert [(n, t) for n, t in _lib.VocProbeArgs._fields_] == want
    enum = re.search(r"enum \{([^}]*AGPT_VC_CF_TO_CL[^}]*)\}", _header(), re.S).group(1)
    names = [e.split("=")[0].strip() for e in enum.split(",") if e.strip()]
    assert names == ["AGPT_VC_" + n for n in _lib.VC_OPS]
    assert "AGPT_VC_CF_TO_CL = 0" in enum and enum.count("=") == 1


def test_an_probe_args_mirror_the_header():
    """_lib.AnProbeArgs has the fields of agpt_an_probe_args in the header's order and C types, and _lib.AN_OPS lists
    the AGPT_AN_* selectors in the enum's order (a mismatch would run another kernel or shift its arguments)."""
    from audiogpt_b200 import _lib
    want = _header_struct_fields("agpt_an_probe_args")
    assert [(n, t) for n, t in _lib.AnProbeArgs._fields_] == want
    enum = re.search(r"enum \{([^}]*AGPT_AN_LASS_AFFINE[^}]*)\}", _header(), re.S).group(1)
    names = [e.split("=")[0].strip() for e in enum.split(",") if e.strip()]
    assert names == ["AGPT_AN_" + n for n in _lib.AN_OPS]
    assert "AGPT_AN_LASS_AFFINE = 0" in enum and enum.count("=") == 1
