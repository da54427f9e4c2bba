"""CPU oracle of FrozenCLAPEmbedder.encode after tokenization (text_to_audio/Make_An_Audio/ldm/modules/encoders/
modules.py:205-212): HF BertModel called with input_ids only (no attention mask: every position attends to every
position, padding included; token type 0), then CLAP's Projection (ldm/modules/encoders/CLAP/clap.py:8-20, dropout
off).  Restated with torch CPU ops from a state dict in the layout of audiogpt_b200.specs.clap_param_shapes; it does
not use transformers."""
import math

import torch
import torch.nn.functional as F


def clap_encode(sd, cfg, input_ids):
    """input_ids [N, L] integer -> z [N, L, d_proj] (fp32, CPU)"""
    ids = torch.as_tensor(input_ids).long().cpu()
    N, L = ids.shape
    H, nh = int(cfg["hidden_size"]), int(cfg["num_heads"])
    dh = H // nh
    eps = float(cfg["layer_norm_eps"])
    b = "caption_encoder.base."
    w = lambda k: sd[b + k].float()   # noqa: E731

    def ln(x, p, e):
        return F.layer_norm(x, (x.shape[-1],), w(p + ".weight"), w(p + ".bias"), e)

    x = w("embeddings.word_embeddings.weight")[ids] + w("embeddings.token_type_embeddings.weight")[0]
    x = x + w("embeddings.position_embeddings.weight")[:L]
    x = ln(x, "embeddings.LayerNorm", eps)
    for i in range(int(cfg["num_layers"])):
        p = f"encoder.layer.{i}."
        q, k, v = (F.linear(x, w(p + f"attention.self.{n}.weight"), w(p + f"attention.self.{n}.bias"))
                   .view(N, L, nh, dh).transpose(1, 2) for n in ("query", "key", "value"))
        a = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh), dim=-1) @ v
        a = a.transpose(1, 2).reshape(N, L, H)
        x = ln(F.linear(a, w(p + "attention.output.dense.weight"), w(p + "attention.output.dense.bias")) + x,
               p + "attention.output.LayerNorm", eps)
        h = F.gelu(F.linear(x, w(p + "intermediate.dense.weight"), w(p + "intermediate.dense.bias")))
        x = ln(F.linear(h, w(p + "output.dense.weight"), w(p + "output.dense.bias")) + x, p + "output.LayerNorm", eps)
    q = "caption_encoder.projection."
    e1 = F.linear(x, sd[q + "linear1.weight"].float())
    e2 = F.linear(F.gelu(e1), sd[q + "linear2.weight"].float())
    return F.layer_norm(e1 + e2, (e1.shape[-1],), sd[q + "layer_norm.weight"].float(), sd[q + "layer_norm.bias"].float(),
                        float(cfg["proj_layer_norm_eps"]))
