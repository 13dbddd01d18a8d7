"""Host loop vs device walk of FasterSparseEngine's grouped zoom-in levels (FasterSparseEngine(device_walk=...)).

The BASELINE.json configs[4] workload at N = 1, as `bench.py --config 5` runs it (tools/engine_bench.py): a synthetic
1024 x 1024 pair, the fixture weights, FasterSparseEngine(model, 32, mode='tile'), 6826 forced queries a -> b, back b -> a
from the answers, 2048 correspondences kept by cycle error, zooms np.linspace(0.5, 0.0625, 4).  The two settings run
alternated, `--repeats` times after one warm-up of each.  Reported medians: the whole call (host clock around work that
ends in a device synchronise) and the grouped levels alone (from the end of gen_tasks to the start of the single-query
fallback, both passes of the call).  The correspondences of the two settings are
checked to be identical, and the GPU's name, power limit and clocks are read in the same run.  Writes one JSON line to
stdout and to --out.
    python tools/grouped_walk_bench.py --out /tmp/grouped_walk_bench.json
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
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "grouped_walk_bench measures on the GPU"
    from cotr_b200.inference.sparse_engine import FasterSparseEngine
    from cotr_b200.utils.utils import fix_randomness
    from tools.engine_bench import _model, _pair, _queries, forced_cycle_consistency

    model = _model(torch.device("cuda", 0))
    img_a, img_b = _pair()
    queries = _queries(int(2048 / 0.3))

    def run(walk):
        """-> (correspondences, ms in the grouped levels, printed lines)"""
        eng = FasterSparseEngine(model, 32, mode='tile', device_walk=walk)
        grouped = []
        gen, single = eng.gen_tasks, eng._single_query_loop

        def gen_tasks(*a, **k):
            tasks = gen(*a, **k)
            torch.cuda.synchronize()
            grouped.append(-time.perf_counter())
            return tasks

        def single_query_loop(tasks, max_corrs, zoom=None):
            if zoom is not None:            # the fallback right after the grouped levels
                torch.cuda.synchronize()
                grouped[-1] += time.perf_counter()
            return single(tasks, max_corrs, zoom)

        eng.gen_tasks, eng._single_query_loop = gen_tasks, single_query_loop
        fix_randomness(0)
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            corr, _ = forced_cycle_consistency(eng, img_a, img_b, queries, 2048)
        return corr, sum(grouped) * 1e3, out.getvalue()

    result = {"gpu": gpu_info(), "repeats": args.repeats, "workload": "configs[4] at N = 1: 1024 x 1024, batch 32, tile, "
              "6826 forced queries, cycle consistency, 2048 correspondences, zooms linspace(0.5, 0.0625, 4)"}
    times = {False: [], True: []}
    outs = {}
    for rep in range(args.repeats + 1):
        for walk in (False, True):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            corr, grouped_ms, printed = run(walk)
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            outs[walk] = (corr, printed)
            if rep > 0:
                times[walk].append((wall, grouped_ms))
            print(f"rep {rep} {'device_walk' if walk else 'host_loop'}: {wall:.1f} ms, grouped levels {grouped_ms:.1f} ms",
                  file=sys.stderr, flush=True)
    assert np.array_equal(outs[False][0], outs[True][0]) and outs[False][1] == outs[True][1]
    result["correspondences"] = int(outs[True][0].shape[0])
    result["grouped_batches_per_call"] = outs[True][1].count("solved ")
    for walk, key in ((False, "host_loop"), (True, "device_walk")):
        t = np.array(times[walk])
        result[key] = {"wall_ms_median": float(np.median(t[:, 0])), "grouped_ms_median": float(np.median(t[:, 1])),
                       "wall_ms_all": [round(float(v), 1) for v in t[:, 0]], "grouped_ms_all": [round(float(v), 1) for v in t[:, 1]]}
    result["speedup_wall"] = result["host_loop"]["wall_ms_median"] / result["device_walk"]["wall_ms_median"]
    result["speedup_grouped"] = result["host_loop"]["grouped_ms_median"] / result["device_walk"]["grouped_ms_median"]
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
