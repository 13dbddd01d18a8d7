"""Generate tests/golden/attn_b2_q100.npz from the REAL reference (run in the authoring container only).

    python -m oracle.make_attention_golden            # needs /root/reference

The unmodified reference model (oracle/ref_shim.py) runs the model_b2_q100 fixture on CPU in fp32 and in fp64 with a
forward hook on each of its 12 nn.MultiheadAttention modules that keeps output[1], the head-averaged attention map.
To keep the file small only sampled rows are stored: one row per image pair of encoder layers 0 and 5 and of
decoder layers 0, 3 and 5.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)

from oracle import attention_oracle, fixtures, ref_shim  # noqa: E402

PARAMS = (0, 3.0, 1.35, 2, 2, 100)           # model_b2_q100: (weight_seed, qk_gain, head_gain, input_seed, batch, n_queries)
LAYERS = (0, 5, 6, 9, 11)                     # index in the call order: encoder 0..5, decoder 0..5
ROWS = ((137, 402), (137, 402), (17, 83), (17, 83), (17, 83))   # sampled query row of pair 0 / pair 1, per stored layer


def _reference_maps(model, img, queries):
    maps = []
    t = model.transformer
    mods = [t.encoder.layers[l].self_attn for l in range(6)] + [t.decoder.layers[l].multihead_attn for l in range(6)]
    handles = [m.register_forward_hook(lambda m_, i_, o_: maps.append(o_[1].detach().clone())) for m in mods]
    try:
        model(img, queries)
    finally:
        for h in handles:
            h.remove()
    assert len(maps) == 12
    return maps


def _sample(maps):
    return np.stack([np.stack([maps[li][b, ROWS[n][b]].numpy() for b in range(2)]) for n, li in enumerate(LAYERS)])


def main():
    torch.set_grad_enabled(False)
    wseed, qk, hg, iseed, b, q = PARAMS
    sd = fixtures.make_state_dict(wseed, qk, hg)
    img, queries = fixtures.make_inputs(iseed, b, q)
    model = ref_shim.build_reference_model(sd)
    ref32 = _reference_maps(model, torch.from_numpy(img), torch.from_numpy(queries))
    ref64 = _reference_maps(model.double(), torch.from_numpy(img).double(), torch.from_numpy(queries).double())
    _, o64 = attention_oracle.forward(sd, img, queries, torch.float64)
    _, o32 = attention_oracle.forward(sd, img, queries, torch.float32)
    for n, (a, b_, c, d) in enumerate(zip(ref64, o64, ref32, o32)):
        print(f"map {n:2d}: |oracle64-ref64| {(a - b_).abs().max().item():.2e}  |oracle32-ref32| {(c - d).abs().max().item():.2e}  "
              f"|ref32-ref64| {(c.double() - a).abs().max().item():.2e}")
    np.savez_compressed(
        os.path.join(REPO, "tests", "golden", "attn_b2_q100.npz"),
        params=np.array(PARAMS, dtype=np.float64), layers=np.array(LAYERS, dtype=np.int64), rows=np.array(ROWS, dtype=np.int64),
        ref_fp32=_sample(ref32).astype(np.float32), ref_fp64=_sample(ref64).astype(np.float64),
    )


if __name__ == "__main__":
    main()
