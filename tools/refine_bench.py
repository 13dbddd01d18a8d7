"""Host loop vs device walk of SparseEngine's single-query zoom-in loop (SparseEngine(device_walk=...)).

Two workloads on a synthetic 1024 x 1024 pair with the fixture weights:
  forced:  2048 forced queries, 4 zoom levels (np.linspace(0.5, 0.0625, 4)), batch 32 - the loop alone, on fresh tasks;
  demo:    the demo_single_pair call - cotr_corr_multiscale_with_cycle_consistency, max_corrs = 100, same zooms, batch 32,
           1000 query points, on weights whose last layer answers near the crop centre (the fixture weights' answers
           leave the image, and the demo's filters would keep nothing).
Each is run with the two settings alternated, `--repeats` times after one warm-up of each; the medians of the wall time
(host clock around work that ends in a device synchronise) and of the CUDA-event time between the same two points are
reported, with the GPU's name, power limit and clocks read in the same run.  The results of the two settings are checked
to be identical.  Writes one JSON line to stdout and to --out.
    python tools/refine_bench.py --out /tmp/refine_bench.json
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:    # the numbers stay meaningful only with it: report why it is missing
        out = f"nvidia-smi unavailable: {e}"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "refine_bench measures on the GPU"
    from cotr_b200.inference.refinement_task import RefinementTask
    from cotr_b200.inference.sparse_engine import SparseEngine
    from cotr_b200.models import build_model
    from cotr_b200.utils.utils import fix_randomness
    from oracle import fixtures
    from oracle.fake_model import synthetic_image

    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in fixtures.make_state_dict(0).items()})
    model = model.cuda().eval()
    img_a, img_b = synthetic_image(61, 1024, 1024), synthetic_image(62, 1024, 1024)
    zooms = np.linspace(0.5, 0.0625, 4)
    rs = np.random.RandomState(0)
    loc_from = rs.uniform(0, 1024, (2048, 2))
    loc_to = np.clip(loc_from + rs.normal(0, 20, (2048, 2)), 0, 1023)

    def forced(walk):
        tasks = [RefinementTask(img_a, img_b, f.copy(), t.copy(), 1.0, 1.0, 1, zooms) for f, t in zip(loc_from, loc_to)]
        SparseEngine(model, 32, device_walk=walk)._single_query_loop(tasks, len(tasks))
        return np.array([np.concatenate(t.loc_history) for t in tasks])

    # The demo's cycle-consistency filter keeps nothing with the fixture weights: its call runs on weights whose last
    # layer answers near the crop centre (as tests/test_refine_gpu.py does), with 1000 query points.
    centred = {k: v.copy() for k, v in fixtures.make_state_dict(0).items()}
    centred["corr_embed.layers.2.weight"] *= 0.01
    centred["corr_embed.layers.2.bias"][:] = (0.75, 0.5)
    demo_model = build_model(None)
    demo_model.load_state_dict({k: torch.from_numpy(v) for k, v in centred.items()})
    demo_model = demo_model.cuda().eval()
    demo_q = rs.uniform(8, 1016, (1000, 2))

    def demo(walk):
        fix_randomness(0)
        return SparseEngine(demo_model, 32, device_walk=walk).cotr_corr_multiscale_with_cycle_consistency(
            img_a, img_b, zooms, 1, max_corrs=100, queries_a=demo_q.copy())

    result = {"gpu": gpu_info(), "repeats": args.repeats}
    for name, fn in (("forced_2048x4", forced), ("demo_single_pair", demo)):
        times = {False: [], True: []}
        outs = {}
        for rep in range(args.repeats + 1):
            for walk in (False, True):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record()
                with contextlib.redirect_stdout(io.StringIO()):
                    outs[walk] = fn(walk)
                e1.record()
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                if rep > 0:
                    times[walk].append((wall * 1e3, e0.elapsed_time(e1)))
                print(f"{name} rep {rep} {'device_walk' if walk else 'host_loop'}: {wall * 1e3:.1f} ms", file=sys.stderr, flush=True)
        assert np.array_equal(outs[False], outs[True]), name
        row = {}
        for walk, key in ((False, "host_loop"), (True, "device_walk")):
            t = np.array(times[walk])
            row[key] = {"wall_ms_median": float(np.median(t[:, 0])), "event_ms_median": float(np.median(t[:, 1])),
                        "wall_ms_all": [round(float(v), 2) for v in t[:, 0]]}
        row["speedup_wall"] = row["host_loop"]["wall_ms_median"] / row["device_walk"]["wall_ms_median"]
        result[name] = row
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
