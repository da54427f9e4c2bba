"""CLAP text encoder (FrozenCLAPEmbedder) on the GPU through the C ABI, against the reference fixtures
(tests/golden/make_golden_clap.py) and the CPU oracle.  Stated tolerance: rel-RMSE <= 1e-4 on z; after DDIM <= 1e-3.
Also the T2A chain from token ids to the sampled latent: CLAP conditioning, then DDIM with classifier-free guidance."""
import ctypes as C

import numpy as np
import pytest
import torch

from audiogpt_b200 import _lib, paramtree, specs
from audiogpt_b200.ldm.modules.encoders.modules import FrozenCLAPEmbedder
from conftest import load_golden, rel_rmse
from oracle import clap_ref

pytestmark = pytest.mark.gpu
SEED = 7070
_SD = {}


def weights(cfg):
    key = cfg["hidden_size"]
    if key not in _SD:
        _SD[key] = specs.synth_clap(cfg, SEED)
    return _SD[key]


def build(cfg, tokenizer=None):
    m = FrozenCLAPEmbedder.from_config(cfg, tokenizer=tokenizer, max_length=cfg["max_length"])
    m.load_state_dict(weights(cfg), strict=True)
    return m.eval().to("cuda")


class StubTokenizer:
    """bert-base-uncased's row layout for fixed prompts: [CLS] ids [SEP], truncated to max_length, zero-padded to it"""

    def __init__(self, table):
        self.table = table

    def __call__(self, text, truncation=True, max_length=77, padding="max_length", return_tensors="pt", **kw):
        rows = []
        for t in [text] if isinstance(text, str) else text:
            body = self.table[t][:max_length - 2]
            rows.append([101] + body + [102] + [0] * (max_length - 2 - len(body)))
        return {"input_ids": torch.tensor(rows, dtype=torch.long)}


def test_small_fixture():
    g = load_golden("clap_small")
    m = build(specs.CLAP_SMALL)
    for L in (77, 20):
        ids = torch.tensor(g[f"ids{L}"])
        z = m.encode_ids(ids.cuda()).cpu()
        ref = clap_ref.clap_encode(weights(specs.CLAP_SMALL), specs.CLAP_SMALL, ids)
        e_fix, e_or = rel_rmse(z, g[f"z{L}"]), rel_rmse(z, ref)
        print(f"clap small L={L}: rel-RMSE vs reference {e_fix:.3e}, vs oracle {e_or:.3e}")
        assert z.shape == (4, L, 48) and e_fix <= 1e-4 and e_or <= 1e-4


def _base_case():
    """T2A's two calls at the shipped shape (3 x [""] then 3 x [prompt]): every row against the stored distinct rows
    and the oracle; the three identical rows of a call come out equal."""
    g = load_golden("clap_base")
    m = build(specs.CLAP_BASE)
    ids = torch.tensor(g["ids"])
    ref = clap_ref.clap_encode(weights(specs.CLAP_BASE), specs.CLAP_BASE, ids)
    for i in range(2):
        z = m.encode_ids(ids[i:i + 1].repeat(3, 1).cuda()).cpu()
        assert z.shape == (3, 77, 1024)
        assert torch.equal(z[0], z[1]) and torch.equal(z[0], z[2])
        e_fix, e_or = rel_rmse(z[0], g["z"][i]), rel_rmse(z[0], ref[i])
        print(f"clap base call {i}: rel-RMSE vs reference {e_fix:.3e}, vs oracle {e_or:.3e}")
        assert e_fix <= 1e-4 and e_or <= 1e-4


def test_base_fixture():
    _base_case()


def test_base_fp32_gemms():
    """the base case again with every GEMM on the fp32-FMA kernel"""
    L = _lib.lib()
    _lib.check(L.agpt_set_tensor_cores(0))
    try:
        _base_case()
    finally:
        _lib.check(L.agpt_set_tensor_cores(1))


def test_batch_independence():
    """each row alone gives what it gives inside the batch (no row reads another's: attention stays per sequence)"""
    g = load_golden("clap_small")
    m = build(specs.CLAP_SMALL)
    ids = torch.tensor(g["ids77"]).cuda()
    both = m.encode_ids(ids)
    for i in range(ids.shape[0]):
        one = m.encode_ids(ids[i:i + 1])
        assert torch.allclose(one[0], both[i], atol=1e-5, rtol=1e-4), i


@pytest.mark.parametrize("L", [1, 20, 80])
def test_single_sequence_lengths(L):
    cfg = specs.CLAP_SMALL
    m = build(cfg)
    ids = torch.randint(0, cfg["vocab_size"], (1, L), generator=torch.Generator().manual_seed(L))
    z = m.encode_ids(ids.cuda()).cpu()
    assert z.shape == (1, L, cfg["d_proj"])
    e = rel_rmse(z, clap_ref.clap_encode(weights(cfg), cfg, ids))
    print(f"clap small N=1 L={L}: rel-RMSE vs oracle {e:.3e}")
    assert e <= 1e-4


def test_bad_inputs_raise():
    cfg = specs.CLAP_SMALL
    m = build(cfg)
    ok = torch.ones((2, 8), dtype=torch.long, device="cuda")
    for bad in (cfg["vocab_size"], -1):
        ids = ok.clone()
        ids[1, 3] = bad
        with pytest.raises(ValueError, match="token ids"):
            m.encode_ids(ids)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        m.encode_ids(torch.ones((1, cfg["max_position_embeddings"] + 1), dtype=torch.long, device="cuda"))
    with pytest.raises(ValueError, match="integer"):
        m.encode_ids(ok.float())
    with pytest.raises(RuntimeError, match="CUDA only"):
        m.encode_ids(ok.cpu())
    cpu = FrozenCLAPEmbedder.from_config(cfg, tokenizer=StubTokenizer({"": []}), device="cpu")
    with pytest.raises(RuntimeError, match="CUDA only"):
        cpu.encode([""])


def test_encode_text_equals_encode_ids():
    cfg = specs.CLAP_SMALL
    table = {"": [], "a dog barks": [7, 300, 41], "thunder": [999, 5]}
    tok = StubTokenizer(table)
    m = build(cfg, tokenizer=tok)
    texts = list(table)
    z = m.encode(texts)
    assert z.device.type == "cuda" and z.shape == (3, cfg["max_length"], cfg["d_proj"])
    assert torch.equal(z, m.encode_ids(tok(texts, max_length=cfg["max_length"])["input_ids"].cuda()))


def test_rebuild_after_weight_edit_and_create_checks_weight_count():
    """the shared engine lifecycle: unchanged weights keep the handle, an in-place edit reaches the next output; a wrong
    weight count is rejected without a handle"""
    m = build(specs.CLAP_SMALL)
    ids = torch.tensor(load_golden("clap_small")["ids20"]).cuda()
    z0 = m.encode_ids(ids).clone()
    h0 = m._h.value
    assert h0 and torch.equal(m.encode_ids(ids), z0) and m._h.value == h0
    with torch.no_grad():
        paramtree.get_tensor(m, "caption_encoder.projection.layer_norm.bias").add_(0.5)
    z1 = m.encode_ids(ids)
    assert torch.allclose(z1, z0 + 0.5, atol=1e-5)
    ws = [paramtree.get_tensor(m, k) for k in m._shapes]
    cfg = _lib.ClapConfig(**m.cfg)
    L = _lib.lib()
    for w, msg in ((ws[:-1], b"too few weight arrays"), (ws + ws[-1:], b"weight array count does not match the config")):
        arr, keep = _lib.host_weight_array(w)
        h = C.c_void_p()
        rc = L.agpt_clap_create(C.byref(cfg), arr, len(keep), torch.cuda.current_device(), C.byref(h))
        assert rc != 0 and msg in L.agpt_last_error(), L.agpt_last_error()
        assert not h.value


def test_t2a_chain_small():
    """T2A on the engine from token ids: CLAP_SMALL encodes uc = 2 x [""] and c = 2 prompts (get_learned_conditioning),
    then DDIMSampler.sample runs DDIM-10 with CFG 1.5 on UNET_SMALL, whose context_dim is CLAP_SMALL's d_proj.
    Compared with clap_ref + the LDM oracle."""
    from audiogpt_b200.ldm.models.diffusion.ddim import DDIMSampler, LatentDiffusionShim
    from audiogpt_b200.ldm.modules.diffusionmodules.openaimodel import UNetModel
    from oracle import ldm_ref as lr
    ccfg, ucfg = specs.CLAP_SMALL, specs.UNET_SMALL
    assert ccfg["d_proj"] == ucfg["context_dim"]
    table = {"": [], "a dog barks while birds sing": [212, 17, 640, 99, 903, 5], "rain on a tin roof": [77, 410, 3, 958]}
    tok = StubTokenizer(table)
    clap = build(ccfg, tokenizer=tok)
    prompts = ["a dog barks while birds sing", "rain on a tin roof"]
    uc, c = clap.encode(2 * [""]), clap.encode(prompts)
    usd = specs.synth_unet(ucfg, 3030)
    u = UNetModel(image_size=32, use_checkpoint=True, **ucfg)
    u.load_state_dict(usd, strict=True)
    smp = DDIMSampler(LatentDiffusionShim(u.eval().cuda()).cuda())
    xT = torch.tensor(np.random.RandomState(55).randn(2, 4, 6, 10), dtype=torch.float32)
    z, _ = smp.sample(S=10, batch_size=2, shape=(4, 6, 10), conditioning=c, verbose=False, x_T=xT.cuda(), eta=0.0,
                      unconditional_guidance_scale=1.5, unconditional_conditioning=uc)
    csd = weights(ccfg)
    rc = clap_ref.clap_encode(csd, ccfg, tok(prompts, max_length=77)["input_ids"])
    ruc = clap_ref.clap_encode(csd, ccfg, tok(2 * [""], max_length=77)["input_ids"])
    assert rel_rmse(c.cpu(), rc) <= 1e-4 and rel_rmse(uc.cpu(), ruc) <= 1e-4
    ref = lr.ddim_sample(lambda a, t, cc: lr.unet_forward(usd, ucfg, a, t, cc), lr.ldm_schedule()["alphas_cumprod"], 10,
                         xT, rc, ruc, 1.5)
    e = rel_rmse(z.cpu(), ref)
    print(f"T2A chain (CLAP -> DDIM-10 + CFG 1.5): latent rel-RMSE vs oracle {e:.3e}")
    assert e <= 1e-3
