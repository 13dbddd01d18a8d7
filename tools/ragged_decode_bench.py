"""Decoding a different number of queries per pair: one ragged call against padding and against one call per pair.

Setup: 8 random images go through the backbone once (encode_images); a 16-pair context of random ordered pairs of them
is built from those cached features (encode_context_pairs).  Pair p asks Q_p queries, drawn once from a seeded
log-uniform distribution over [64, 4096] (the keypoint counts of an image set differ that way).  Three arms decode the
same queries on the GPU:
  (a) padded:   one cotr_decode of the (16, max Q_p, 2) block, every pair zero-padded to the largest count;
  (b) ragged:   one cotr_decode_ragged of the packed (sum Q_p, 2) rows;
  (c) per pair: 16 cotr_decode calls, each on a one-pair context of the same pair (built beforehand, not timed).
Each call is timed with CUDA events after warm-up and after the L2 is flushed; the arms alternate and the median is
reported as ms per call and as real query points per second (padding rows do not count).  The predictions of the real
rows must agree between the arms within 2e-4.  The card's name and power limit are read in the same run.

    python tools/ragged_decode_bench.py [--repeats 20] [--warmup 3] [--seed 0] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

PAIRS = 16
IMAGES = 8
QMIN, QMAX = 64, 4096
AGREE_TOL = 2e-4


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from cotr_b200.models import build_model
    from cotr_b200.utils import synthetic

    assert torch.cuda.is_available(), "ragged_decode_bench needs the GPU"
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in synthetic.make_state_dict(0).items()})
    model = model.cuda().eval()
    nat = model.native()
    rs = np.random.RandomState(args.seed)
    images = torch.from_numpy(rs.standard_normal((IMAGES, 3, 256, 256)).astype(np.float32)).cuda()
    pairs = []
    while len(pairs) < PAIRS:
        i, j = rs.randint(IMAGES, size=2)
        if i != j:
            pairs.append((int(i), int(j)))
    counts = np.exp(rs.uniform(np.log(QMIN), np.log(QMAX), PAIRS)).astype(np.int64)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    R, Qmax = int(offsets[-1]), int(counts.max())
    qs = [torch.from_numpy(rs.uniform(0, 1, (int(n), 2)).astype(np.float32)).cuda() for n in counts]
    packed = torch.cat(qs).contiguous()
    padded = torch.zeros((PAIRS, Qmax, 2), dtype=torch.float32, device="cuda")
    for p, q in enumerate(qs):
        padded[p, :q.shape[0]] = q

    feats = model.encode_images(images)
    ctx = model.encode_context_pairs(feats, pairs)
    singles = [model.encode_context_pairs(feats, [pr]) for pr in pairs]
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")

    def timed(fn):
        flush.zero_()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    def arm_padded():
        pred = nat.decode(ctx.native, padded)
        return torch.cat([pred[p, :int(n)] for p, n in enumerate(counts)])

    def arm_ragged():
        return nat.decode_ragged(ctx.native, packed, offsets)

    def arm_per_pair():
        return torch.cat([nat.decode(c.native, q[None])[0] for c, q in zip(singles, qs)])

    arms = (("padded", arm_padded), ("ragged", arm_ragged), ("per_pair", arm_per_pair))
    launches = {}
    for name, fn in arms:
        for _ in range(args.warmup):
            fn()
        if name != "per_pair":
            launches[name] = nat.last_launch_count()
    torch.cuda.synchronize()
    preds = {name: fn() for name, fn in arms}
    diffs = {f"{a}_vs_ragged": (preds[a] - preds["ragged"]).abs().max().item() for a in ("padded", "per_pair")}
    times = {name: [] for name, _ in arms}
    for _ in range(args.repeats):
        for name, fn in arms:
            times[name].append(timed(fn)[0])

    result = dict(card=card(), torch_device=torch.cuda.get_device_name(), pairs=PAIRS, counts=counts.tolist(),
                  real_rows=R, padded_rows=PAIRS * Qmax, repeats=args.repeats, launches=launches, max_abs_diff=diffs)
    for name, _ in arms:
        ms = float(np.median(times[name]))
        result[name] = dict(ms_per_call=ms, ms_min_max=(float(np.min(times[name])), float(np.max(times[name]))),
                            real_query_points_per_s=R / (ms * 1e-3))
    print(f"card: {result['card']}")
    print(f"{PAIRS} pairs, {R} real query rows (padded block: {PAIRS * Qmax} rows, largest count {Qmax})")
    for name, _ in arms:
        r = result[name]
        print(f"  {name:9s} {r['ms_per_call']:.3f} ms per call ({r['ms_min_max'][0]:.3f} .. {r['ms_min_max'][1]:.3f}), "
              f"{r['real_query_points_per_s'] / 1e6:.2f} M real query points/s")
    print("  max |diff| of the real rows: " + ", ".join(f"{k} {v:.2e}" for k, v in diffs.items()), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    bad = {k: v for k, v in diffs.items() if not v < AGREE_TOL}
    assert not bad, f"the arms disagree beyond {AGREE_TOL}: {bad}"


if __name__ == "__main__":
    main()
