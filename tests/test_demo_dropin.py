"""BASELINE.json configs[0]: the call sequence of the reference's `demo_single_pair.py` through the alias package.

The script's imports (`from COTR.models import build_model`, `from COTR.inference.sparse_engine import SparseEngine`,
`from COTR.utils import utils` ...) bind to the alias package `COTR/` -> `cotr_b200`; the test below makes the same
calls in the same order on the GPU, with the changes SURVEY.md section 8(d) prescribes for random weights.
"""
import os
import sys

import numpy as np
import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_demo_call_sequence_native_gpu(tmp_path, capsys, built_lib):
    """What `demo_single_pair.py:25-45` does, with the changes SURVEY.md section 8(d) prescribes for random weights:
    synthetic images instead of the sample pair and 100 FORCED queries (`cotr_corr_multiscale(..., queries_a=q, force=True)`), so every query comes back.  Everything
    goes through the alias package `COTR`, as in the script: build_model -> cuda -> checkpoint file -> safe_load_weights ->
    SparseEngine(model, 32, mode='tile') -> visualize_corrs -> triangulate_corr (CUDA rasteriser) -> cv2.remap."""
    import cv2
    sys.path.insert(0, REPO)
    from COTR.utils import utils
    from COTR.models import build_model
    from COTR.inference.inference_helper import triangulate_corr
    from COTR.inference.sparse_engine import SparseEngine
    from cotr_b200.utils import synthetic

    utils.fix_randomness(0)
    torch.set_grad_enabled(False)
    ckpt = tmp_path / "checkpoint.pth.tar"
    torch.save({"model_state_dict": {k: torch.from_numpy(v) for k, v in synthetic.make_state_dict(0).items()}}, ckpt)
    model = build_model(None).cuda()
    utils.safe_load_weights(model, torch.load(ckpt, map_location='cpu')['model_state_dict'])
    model = model.eval()
    img_a = synthetic.synthetic_image(61, 783, 1064)          # the shapes of cathedral_1.jpg / cathedral_2.jpg
    img_b = synthetic.synthetic_image(62, 1053, 689)
    rs = np.random.RandomState(0)
    queries = np.stack([rs.uniform(0, img_a.shape[1], 100), rs.uniform(0, img_a.shape[0], 100)], axis=1)
    engine = SparseEngine(model, 32, mode='tile')
    corrs = engine.cotr_corr_multiscale(img_a, img_b, np.linspace(0.5, 0.0625, 4), 1, max_corrs=100, queries_a=queries, force=True)
    assert corrs.shape == (100, 4) and np.isfinite(corrs).all()
    assert np.allclose(np.sort(corrs[:, 0]), np.sort(queries[:, 0]))            # every forced query came back
    canvas = utils.visualize_corrs(img_a, img_b, corrs)
    assert canvas.shape == (1053, 1064 + 689, 3)
    dense = triangulate_corr(corrs, img_a.shape, img_b.shape)
    assert dense.shape == (783, 1064, 2) and dense.dtype == np.float32 and (dense != 0).any()
    warped = cv2.remap(img_b, dense[..., 0].astype(np.float32), dense[..., 1].astype(np.float32), interpolation=cv2.INTER_LINEAR,
                       borderMode=cv2.BORDER_CONSTANT)
    assert warped.shape == img_a.shape
    assert "weights safely loaded" in capsys.readouterr().out
