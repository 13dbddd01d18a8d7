"""'stretching' mode's dense first guess on the device against the host path, in the two demo calls that use that mode.

Workloads (synthetic images at the demos' sizes, the fixture weights, batch 32, zooms np.linspace(0.5, 0.0625, 4),
SparseEngine(model, 32, mode='stretching', device_walk=True)):
  * homography: a 4032 x 3024 and a 1920 x 1080 image (W x H), the 4 image corners of the first as float32 queries, forced
    (demo_homography.py's call);
  * face: 794 x 688 and 928 x 688 images, 68 landmark-like points, unforced (demo_face.py's call).
Arms: inference_helper.DEVICE_STRETCH = True (stretch, dense pass and resize back on the device, four maps copied back)
and False (PIL stretch, dense pass, maps to the host, float_image_resize), alternated, `--repeats` times after one warm-up
of each.  Reported per arm: medians of the whole call and of its dense first guess (host clock around
SparseEngine._dense_first_guess, which ends in a device-to-host copy); the walk is the rest.  The two arms' returns are
checked to be identical, and the GPU's name, power limit and clocks are read in the same run.  Writes one JSON line to
stdout and to --out.
    python tools/stretch_bench.py --out /tmp/stretch_bench.json
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

ZOOMS = np.linspace(0.5, 0.0625, 4)
BATCH = 32


def workloads():
    from cotr_b200.utils import synthetic
    rs = np.random.RandomState(0)
    paint_1, paint_2 = synthetic.synthetic_image(201, 3024, 4032), synthetic.synthetic_image(202, 1080, 1920)
    corners = np.array([[0, 0], [4032, 0], [4032, 3024], [0, 3024]], dtype=np.float32)
    face_a, face_b = synthetic.synthetic_image(203, 688, 794), synthetic.synthetic_image(204, 688, 928)
    landmarks = np.stack([rs.uniform(250, 550, 68), rs.uniform(150, 550, 68)], axis=1)
    return {
        "homography": lambda e: e.cotr_corr_multiscale(paint_1, paint_2, ZOOMS, 1, queries_a=corners, force=True),
        "face": lambda e: e.cotr_corr_multiscale(face_a, face_b, ZOOMS, 1, max_corrs=68, queries_a=landmarks, force=False),
    }


def run(model, call, device):
    from cotr_b200.inference import inference_helper
    from cotr_b200.inference.sparse_engine import SparseEngine
    inference_helper.DEVICE_STRETCH = device
    eng = SparseEngine(model, BATCH, mode='stretching', device_walk=True)
    dense = []
    real = eng._dense_first_guess

    def timed(img_a, img_b):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = real(img_a, img_b)
        torch.cuda.synchronize()
        dense.append((time.perf_counter() - t0) * 1e3)
        return out
    eng._dense_first_guess = timed
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()), np.errstate(all='ignore'):
        out = call(eng)
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3, sum(dense)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stretch_bench measures on the GPU"
    from cotr_b200.models import build_model
    from cotr_b200.utils import synthetic
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in synthetic.make_state_dict(0).items()})
    model = model.cuda().eval()

    result = {"gpu": gpu_info(), "repeats": args.repeats,
              "workload": "SparseEngine(mode='stretching', device_walk=True), batch 32, zooms linspace(0.5, 0.0625, 4), fixture "
                          "weights; homography: 4032x3024 + 1920x1080, 4 float32 corners, forced; face: 794x688 + 928x688, "
                          "68 points, unforced"}
    for name, call in workloads().items():
        arms = {"device": True, "host": False}
        times = {k: {"wall": [], "dense": []} for k in arms}
        outs = {}
        for rep in range(args.repeats + 1):
            for arm, flag in arms.items():
                outs[arm], wall, dense = run(model, call, flag)
                if rep > 0:
                    times[arm]["wall"].append(wall)
                    times[arm]["dense"].append(dense)
                print(f"{name} rep {rep} {arm}: {wall:.1f} ms (dense first guess {dense:.1f} ms)", file=sys.stderr, flush=True)
        a, b = np.asarray(outs["device"]), np.asarray(outs["host"])
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=True), name
        res = {"corrs": int(a.shape[0])}
        for arm in arms:
            wall, dense = np.median(times[arm]["wall"]), np.median(times[arm]["dense"])
            res[arm] = {"wall_ms_median": round(float(wall), 2), "dense_first_guess_ms_median": round(float(dense), 2),
                        "walk_ms_median": round(float(np.median(np.subtract(times[arm]["wall"], times[arm]["dense"]))), 2),
                        "wall_ms_all": [round(v, 1) for v in times[arm]["wall"]]}
        res["dense_first_guess_speedup"] = res["host"]["dense_first_guess_ms_median"] / res["device"]["dense_first_guess_ms_median"]
        res["wall_speedup"] = res["host"]["wall_ms_median"] / res["device"]["wall_ms_median"]
        result[name] = res
    from cotr_b200.inference import inference_helper
    inference_helper.DEVICE_STRETCH = True
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
