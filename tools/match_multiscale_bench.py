"""match_keypoints_multiscale against the per-pair sequence it replaces, on an image set.

Workload: 4 synthetic images at the sizes of the demo's pair (1033 x 771, 694 x 1061), one more 1033 x 771 and one square
640 x 640, 512 keypoints each from the DISK fixtures (scaled to the image, seeded sub-pixel jitter), all 6 pairs, the
fixture weights, batch 32, zooms np.linspace(0.5, 0.0625, 4).  Arms:
  * per_pair: for every pair SparseEngine(model, 32, mode='tile', device_walk=True).cotr_corr_multiscale(..., force=True)
    in both directions, then mutual_nearest (what a user of demo_guided_matching.py writes for an image set);
  * one_call: cotr_b200.inference.matching.match_keypoints_multiscale.
The arms run alternated, `--repeats` times after one warm-up of each; reported: medians of the whole call (host clock
around work that ends in a device synchronise).  The results of the two arms are checked to be identical (corrs bit for
bit, matches exactly), and the GPU's name, power limit and clocks are read in the same run.  Writes one JSON line to
stdout and to --out.
    python tools/match_multiscale_bench.py --out /tmp/match_multiscale_bench.json
"""
import argparse
import contextlib
import io
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.grouped_walk_bench import gpu_info  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
DISK_A = "disk_kpts_21526113_4379776807.npy"      # image 1033 x 771 (W x H)
DISK_B = "disk_kpts_21126421_4537535153.npy"      # image 694 x 1061
ZOOMS = np.linspace(0.5, 0.0625, 4)
BATCH = 32


def image_set(n_kp=512):
    from cotr_b200.utils import synthetic
    rs = np.random.RandomState(0)
    spec = [(771, 1033, DISK_A, 1.0), (1061, 694, DISK_B, 1.0), (771, 1033, DISK_A, 1.0), (640, 640, DISK_A, 0.6)]
    images, kps = [], []
    for i, (h, w, name, scale) in enumerate(spec):
        images.append(synthetic.synthetic_image(100 + i, h, w))
        k = np.load(os.path.join(GOLDEN, name))[:n_kp] * np.float32(scale)
        k = k + rs.uniform(-0.5, 0.5, k.shape)
        kps.append(np.clip(k, 0, [w - 1, h - 1]).astype(np.float32))
    return images, kps


def per_pair(model, images, kps, pairs):
    from cotr_b200.inference.matching import mutual_nearest
    from cotr_b200.inference.sparse_engine import SparseEngine
    eng = SparseEngine(model, BATCH, mode='tile', device_walk=True)
    out = []
    for a, b in pairs:
        c_ab = eng.cotr_corr_multiscale(images[a], images[b], ZOOMS, 1, max_corrs=len(kps[a]), queries_a=kps[a], force=True)[:, 2:]
        c_ba = eng.cotr_corr_multiscale(images[b], images[a], ZOOMS, 1, max_corrs=len(kps[b]), queries_a=kps[b], force=True)[:, 2:]
        out.append((c_ab, c_ba, mutual_nearest(c_ab, kps[b], c_ba, kps[a])))
    return out


def one_call(model, images, kps, pairs):
    from cotr_b200.inference.matching import match_keypoints_multiscale
    res = match_keypoints_multiscale(model, images, kps, np.array(pairs), ZOOMS, BATCH)
    return [(res.corrs_ab[p].cpu().numpy(), res.corrs_ba[p].cpu().numpy(), res.matches[p].cpu().numpy()) for p in range(len(pairs))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "match_multiscale_bench measures on the GPU"
    from cotr_b200.models import build_model
    from cotr_b200.utils import synthetic
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in synthetic.make_state_dict(0).items()})
    model = model.cuda().eval()
    images, kps = image_set()
    pairs = [(a, b) for a in range(len(images)) for b in range(a + 1, len(images))]

    result = {"gpu": gpu_info(), "repeats": args.repeats, "workload": "4 images (1033x771, 694x1061, 1033x771, 640x640), 512 DISK "
              "keypoints each, all 6 pairs, batch 32, tile, zooms linspace(0.5, 0.0625, 4), fixture weights"}
    arms = {"per_pair": per_pair, "one_call": one_call}
    times = {k: [] for k in arms}
    outs = {}
    for rep in range(args.repeats + 1):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with contextlib.redirect_stdout(io.StringIO()), np.errstate(all='ignore'):
                outs[name] = fn(model, images, kps, pairs)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
            if rep > 0:
                times[name].append(ms)
            print(f"rep {rep} {name}: {ms:.1f} ms", file=sys.stderr, flush=True)
    for (a_ab, a_ba, a_m), (b_ab, b_ba, b_m) in zip(outs["per_pair"], outs["one_call"]):
        assert np.array_equal(a_ab.view(np.int64), b_ab.view(np.int64)) and np.array_equal(a_ba.view(np.int64), b_ba.view(np.int64))
        assert np.array_equal(a_m, b_m)
    result["matches_per_pair"] = [int(len(m)) for _, _, m in outs["one_call"]]
    for name in arms:
        result[name] = {"wall_ms_median": float(np.median(times[name])), "wall_ms_all": [round(v, 1) for v in times[name]]}
    result["speedup"] = result["per_pair"]["wall_ms_median"] / result["one_call"]["wall_ms_median"]
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
