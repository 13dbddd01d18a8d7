"""Matching the keypoints of an image set: one match_keypoints call against the same step built from the existing calls
with the demo's rule on the host.

Setup: 8 random images go through the backbone once (encode_images).  Every image gets 2048 keypoints: the DISK
keypoints of tests/golden (an image of 1033 x 771) with seeded jitter of 1 pixel.  All 28 unordered pairs are matched,
so each call decodes 56 contexts and 114 688 queries and compares 56 x 2048 x 2048 = 235 M candidate distances.  Arms:
  (a) device:  one COTR.match_keypoints call (its one device-to-host copy of the match counts included);
  (b) host:    encode_context_pairs of the same 56 contexts + one ragged decode of oracle-built queries, then per pair
               the oracle's vectorised host rule (pixels, nearest in fp64 by row blocks, mutual) on the copied predictions;
  (c) kernels: the four launches match_keypoints adds (match_queries, match_pixels, nearest, mutual), from the library's
               per-launch profiler in separate calls.
Each call is timed with CUDA events after warm-up and after the L2 is flushed; (a) and (b) alternate and medians are
reported.  The matches of (a) and (b) must be identical.  The card's name and power limit are read in the same run.

    python tools/match_bench.py [--repeats 10] [--warmup 2] [--seed 0] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

IMAGES = 8
SIZE = (1033, 771)          # the image the DISK fixture was detected on
NEW_KERNELS = ("match_queries", "match_pixels", "nearest", "mutual")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from cotr_b200.models import build_model
    from cotr_b200.utils import synthetic
    from oracle import match_oracle as mo

    assert torch.cuda.is_available(), "match_bench needs the GPU"
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in synthetic.make_state_dict(0).items()})
    model = model.cuda().eval()
    nat = model.native()
    rs = np.random.RandomState(args.seed)
    images = torch.from_numpy(rs.standard_normal((IMAGES, 3, 256, 256)).astype(np.float32)).cuda()
    disk = np.load(os.path.join(REPO, "tests", "golden", "disk_kpts_21526113_4379776807.npy"))
    kps = [np.clip(disk + rs.normal(0, 1.0, disk.shape), 0, SIZE).astype(np.float32) for _ in range(IMAGES)]
    sizes = np.array([SIZE] * IMAGES)
    pairs = [(a, b) for a in range(IMAGES) for b in range(a + 1, IMAGES)]
    table = [t for a, b in pairs for t in ((a, b), (b, a))]
    rows = sum(len(kps[l]) for l, _ in table)
    candidates = sum(len(kps[l]) * len(kps[r]) for l, r in table)
    feats = model.encode_images(images)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    host_ms = []

    def arm_device():
        return [m.cpu().numpy() for m in model.match_keypoints(feats, pairs, kps, sizes).matches]

    def arm_host():
        ctx = model.encode_context_pairs(feats, table, reuse=True)
        qs = [torch.from_numpy(mo.queries(kps[l], SIZE)).cuda() for l, _ in table]
        preds = [p.cpu().numpy() for p in model.decode(ctx, qs)["pred_corrs"]]
        t0 = time.perf_counter()
        corrs = [mo.pixels(p, SIZE) for p in preds]
        out = [mo.match_pair(corrs[2 * p], kps[b], corrs[2 * p + 1], kps[a])[2] for p, (a, b) in enumerate(pairs)]
        host_ms.append((time.perf_counter() - t0) * 1e3)
        return out

    def timed(fn):
        flush.zero_()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    arms = (("device", arm_device), ("host", arm_host))
    for _ in range(args.warmup):
        for _, fn in arms:
            fn()
    got = {name: fn() for name, fn in arms}
    identical = all(np.array_equal(x, y) for x, y in zip(got["device"], got["host"]))
    n_matches = int(sum(len(m) for m in got["device"]))
    host_ms.clear()
    times = {name: [] for name, _ in arms}
    for _ in range(args.repeats):
        for name, fn in arms:
            times[name].append(timed(fn)[0])
    kernel_ms = {k: [] for k in NEW_KERNELS}
    for _ in range(args.repeats):
        flush.zero_()
        torch.cuda.synchronize()
        nat.profile_begin(8192)
        model.match_keypoints(feats, pairs, kps, sizes)
        rec = nat.profile_end()
        for k in NEW_KERNELS:
            kernel_ms[k].append(sum(r[4] for r in rec if r[0] == k))

    result = dict(card=card(), torch_device=torch.cuda.get_device_name(), images=IMAGES, pairs=len(pairs), contexts=len(table),
                  keypoints_per_image=len(disk), decoded_queries=rows, candidate_distances=candidates, matches=n_matches,
                  identical_matches=identical, repeats=args.repeats)
    for name, _ in arms:
        result[name] = dict(ms_per_call=float(np.median(times[name])),
                            ms_min_max=(float(np.min(times[name])), float(np.max(times[name]))))
    result["host"]["host_rule_ms"] = float(np.median(host_ms))
    result["kernels_ms"] = {k: float(np.median(v)) for k, v in kernel_ms.items()}
    result["kernels_ms"]["total"] = float(np.median([sum(kernel_ms[k][i] for k in NEW_KERNELS) for i in range(args.repeats)]))
    print(f"card: {result['card']}")
    print(f"{IMAGES} images x {len(disk)} keypoints, {len(pairs)} pairs: {rows} decoded queries, {candidates / 1e6:.0f} M candidate "
          f"distances, {n_matches} mutual matches, identical: {identical}")
    for name, _ in arms:
        r = result[name]
        print(f"  ({'a' if name == 'device' else 'b'}) {name:7s} {r['ms_per_call']:.2f} ms per call "
              f"({r['ms_min_max'][0]:.2f} .. {r['ms_min_max'][1]:.2f})")
    print(f"      host rule alone {result['host']['host_rule_ms']:.1f} ms")
    print("  (c) new launches: " + ", ".join(f"{k} {v:.3f} ms" for k, v in result["kernels_ms"].items()), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    assert identical, "match_keypoints and the host composition disagree"


if __name__ == "__main__":
    main()
