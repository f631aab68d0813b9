"""CPU oracle for the text towers: CLIP.encode_text (openai-CLIP model.py; SLIP/models.py:136-150 has the same structure)
restated in float64 from the checkpoint's tensors.

TEST INFRASTRUCTURE ONLY.  Cross-checked against transformers.CLIPTextModelWithProjection with the same weights
(tests/test_text_tower.py); the GPU tests compare the engine's tower with it.

    x = token_embedding[ids] + positional_embedding
    per block: x = x + out_proj(MHA(ln_1(x)) with the causal mask); x = x + c_proj(QuickGELU(c_fc(ln_2(x))))
    e = ln_final(x)[arange(n), ids.argmax(-1)] @ text_projection
"""
import re

import torch
import torch.nn.functional as F


def shape(sd):
    """(width, layers, context, out_dim) as openai's build_model reads them off the state_dict."""
    layers = len({m.group(1) for k in sd for m in [re.match(r"transformer\.resblocks\.(\d+)\.", k)] if m})
    return sd["token_embedding.weight"].shape[1], layers, sd["positional_embedding"].shape[0], sd["text_projection"].shape[1]


def encode_text(sd, ids, dtype=torch.float64):
    """Un-normalised embeddings [n, D] of token ids [n, T] (any integer array)."""
    W, L, T, _ = shape(sd)
    H = W // 64
    g = {k: torch.as_tensor(v).to(dtype) for k, v in sd.items() if not k.startswith("visual.")}
    ids = torch.as_tensor(ids, dtype=torch.long).reshape(-1, T)
    n = ids.shape[0]
    ln = lambda x, p: F.layer_norm(x, (W,), g[p + ".weight"], g[p + ".bias"], 1e-5)  # noqa: E731
    mask = torch.full((T, T), float("-inf"), dtype=dtype).triu(1)
    x = g["token_embedding.weight"][ids] + g["positional_embedding"]
    for i in range(L):
        p = f"transformer.resblocks.{i}."
        h = ln(x, p + "ln_1")
        qkv = h @ g[p + "attn.in_proj_weight"].T + g[p + "attn.in_proj_bias"]
        q, k, v = (t.reshape(n, T, H, 64).transpose(1, 2) for t in qkv.split(W, dim=-1))
        a = torch.softmax(q @ k.transpose(-1, -2) / 8.0 + mask, dim=-1)
        o = (a @ v).transpose(1, 2).reshape(n, T, W)
        x = x + o @ g[p + "attn.out_proj.weight"].T + g[p + "attn.out_proj.bias"]
        u = ln(x, p + "ln_2") @ g[p + "mlp.c_fc.weight"].T + g[p + "mlp.c_fc.bias"]
        x = x + (u * torch.sigmoid(1.702 * u)) @ g[p + "mlp.c_proj.weight"].T + g[p + "mlp.c_proj.bias"]
    x = ln(x, "ln_final")
    return x[torch.arange(n), ids.argmax(dim=-1)] @ g["text_projection"]


def causal_attention(qkv, B, T, H):
    """softmax(q k^T / 8 + causal mask) v of fp16 qkv [B*T, 3W] (heads 64 wide) in float64 -> [B*T, W]."""
    W = 64 * H
    x = torch.as_tensor(qkv).double().reshape(B, T, 3, H, 64).permute(2, 0, 3, 1, 4)
    mask = torch.full((T, T), float("-inf"), dtype=torch.float64).triu(1)
    a = torch.softmax(x[0] @ x[1].transpose(-1, -2) / 8.0 + mask, dim=-1)
    return (a @ x[2]).transpose(1, 2).reshape(B * T, W)
