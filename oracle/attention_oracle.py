"""Head-averaged attention maps of the CPU restatement (TEST ORACLE - not product code).

The reference calls every ``nn.MultiheadAttention`` of the transformer with ``need_weights=True`` (the default,
COTR/models/transformer.py:149-153 and :192-195), so each call also returns the attention weights averaged over the
8 heads: ``(B, L, 512)`` with value ``mean_h softmax_j(q_h[i] . k_h[j])``.  ``forward`` restates ``cotr_oracle.forward``
stage for stage (same functions, same arithmetic, so the predictions are identical) and keeps those maps.

Pinned against the real reference by oracle/make_attention_golden.py (tests/golden/attn_b2_q100.npz).
"""
import torch
import torch.nn.functional as F

from oracle import cotr_oracle as co


def _mha(q_in, k_in, v_in, sd, prefix, maps):
    """cotr_oracle._mha, also appending the head-averaged weights (B, Lq, Lk) to `maps`."""
    w = sd[prefix + ".in_proj_weight"]
    b = sd[prefix + ".in_proj_bias"]
    d = co.D_MODEL
    q = F.linear(q_in, w[0:d], b[0:d]) * (co.HEAD_DIM ** -0.5)
    k = F.linear(k_in, w[d:2 * d], b[d:2 * d])
    v = F.linear(v_in, w[2 * d:3 * d], b[2 * d:3 * d])
    B, Lq, _ = q.shape
    Lk = k.shape[1]
    q = q.view(B, Lq, co.N_HEAD, co.HEAD_DIM).transpose(1, 2)
    k = k.view(B, Lk, co.N_HEAD, co.HEAD_DIM).transpose(1, 2)
    v = v.view(B, Lk, co.N_HEAD, co.HEAD_DIM).transpose(1, 2)
    attn = torch.softmax(q @ k.transpose(-1, -2), dim=-1)
    maps.append(attn.mean(dim=1))
    o = (attn @ v).transpose(1, 2).reshape(B, Lq, d)
    return F.linear(o, sd[prefix + ".out_proj.weight"], sd[prefix + ".out_proj.bias"])


@torch.no_grad()
def forward(sd, img, queries, dtype=torch.float32):
    """-> (pred (B,Q,2), maps): maps is the list of the 12 head-averaged attention maps in the reference's call order,
    encoder layers 0..5 (B,512,512) then decoder layers 0..5 (B,Q,512)."""
    sd = co.cast_state_dict(sd, dtype)
    img = torch.as_tensor(img).to(dtype)
    q_in = torch.as_tensor(queries).to(dtype)
    B = img.shape[0]
    feat = torch.cat([co.backbone_half(img[..., :co.MAX_SIZE], sd), co.backbone_half(img[..., co.MAX_SIZE:], sd)], dim=-1)
    x = F.conv2d(feat, sd["input_proj.weight"], sd["input_proj.bias"]).flatten(2).transpose(1, 2)
    pos = co.grid_position(dtype)
    qpos = co.lin_sine(q_in.reshape(-1, 2), co.D_MODEL // 4).reshape(B, -1, co.D_MODEL)
    maps = []
    for l in range(co.N_ENC):
        p = f"transformer.encoder.layers.{l}"
        qk = x + pos
        x = co._ln(x + _mha(qk, qk, x, sd, p + ".self_attn", maps), sd, p + ".norm1")
        x = co._ln(x + co._ffn(x, sd, p), sd, p + ".norm2")
    t = torch.zeros_like(qpos)
    kmem = x + pos
    for l in range(co.N_DEC):
        p = f"transformer.decoder.layers.{l}"
        t = co._ln(t + _mha(t + qpos, kmem, x, sd, p + ".multihead_attn", maps), sd, p + ".norm2")
        t = co._ln(t + co._ffn(t, sd, p), sd, p + ".norm3")
    hs = co._ln(t, sd, "transformer.decoder.norm")
    return co.head(hs, sd), maps
