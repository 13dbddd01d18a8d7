"""CPU: the oracle's head-averaged attention maps against the maps the REAL reference's nn.MultiheadAttention modules
return to forward hooks (oracle/make_attention_golden.py -> tests/golden/attn_b2_q100.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import attention_oracle, cotr_oracle, fixtures


def _golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "attn_b2_q100.npz"))
    wseed, qk, hg, iseed, b, q = g["params"]
    sd = fixtures.make_state_dict(int(wseed), float(qk), float(hg))
    img, queries = fixtures.make_inputs(int(iseed), int(b), int(q))
    return g, sd, img, queries


@pytest.mark.parametrize("dtype,key,tol", [(torch.float64, "ref_fp64", 1e-10), (torch.float32, "ref_fp32", 5e-6)],
                         ids=["fp64", "fp32"])
def test_oracle_attention_maps_match_reference(golden_dir, dtype, key, tol):
    g, sd, img, queries = _golden(golden_dir)
    pred, maps = attention_oracle.forward(sd, img, queries, dtype)
    assert len(maps) == 12
    assert all(tuple(m.shape) == (2, 512, 512) for m in maps[:6]) and all(tuple(m.shape) == (2, 100, 512) for m in maps[6:])
    # the restatement with maps computes exactly what the plain oracle computes
    assert torch.equal(pred, cotr_oracle.forward(sd, img, queries, dtype))
    got = np.stack([np.stack([maps[li][b, g["rows"][n][b]].numpy() for b in range(2)]) for n, li in enumerate(g["layers"])])
    assert np.abs(got - g[key]).max() < tol
    assert np.abs(g["ref_fp64"].sum(-1) - 1).max() < 1e-12
