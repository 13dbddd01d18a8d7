"""Matching one image against many, and all ordered pairs of an image set: canvas forward against cached image features.

Two workloads, both at 1024 queries per pair and 8 pairs per batch:
  (a) one query image against 32 database images whose features were computed beforehand (localisation re-ranking).
      Feature arm per step: encode_images(query) + 4 x (encode_context_pairs + decode); the one-off database encode
      is timed on its own.  Canvas arm: 4 x forward of [query | db_i] canvases.
  (b) all 56 ordered pairs of 8 images.  Feature arm per step: encode_images(8) + 7 x (encode_context_pairs + decode).
      Canvas arm: 7 x forward.
Each step is timed with CUDA events, after the L2 is flushed; the arms alternate, and the median step is reported as ms
per pair and query points per second.  The two arms differ only in which images share a backbone pass (a context of
the same halves in the same batch is bitwise the canvas one), so their predictions are checked against the canvas
path's own batch-composition drift, measured in the same run by forwarding every pair alone: they must agree within
2e-4, or within twice that drift where the drift itself exceeds 2e-4 (on an H100 it reached 2.1e-4 in (a) and 2.2e-4
in (b): the maximum over 32 768 and 57 344 query points).
The card's name and power limit are read in the same run.

    python tools/image_pairs_bench.py [--repeats 20] [--warmup 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

Q = 1024
BATCH = 8
AGREE_TOL = 2e-4


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from cotr_b200.models import build_model
    from cotr_b200.models.cotr_model import ImageFeatures
    from cotr_b200.utils import synthetic

    assert torch.cuda.is_available(), "image_pairs_bench needs the GPU"
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in synthetic.make_state_dict(0).items()})
    model = model.cuda().eval()
    rs = np.random.RandomState(7)
    rand = lambda *shape: torch.from_numpy(rs.standard_normal(shape).astype(np.float32)).cuda()
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

    def canvases(images, pairs):
        return torch.stack([torch.cat([images[i], images[j]], dim=-1) for i, j in pairs])

    # (a) one query image against 32 database images
    query_img, db = rand(1, 3, 256, 256), rand(32, 3, 256, 256)
    pairs_a = [(0, 1 + i) for i in range(32)]               # image 0 = the query, 1..32 = the database
    all_a = torch.cat([query_img, db])
    canv_a = [canvases(all_a, pairs_a[k:k + BATCH]).contiguous() for k in range(0, 32, BATCH)]
    uniform = lambda *shape: torch.from_numpy(rs.uniform(0, 1, shape).astype(np.float32)).cuda()
    q_a = [uniform(BATCH, Q, 2) for _ in range(0, 32, BATCH)]

    def canvas_a():
        return [model(c, q)["pred_corrs"] for c, q in zip(canv_a, q_a)]

    db_feat = model.encode_images(db)

    def features_a():
        f = model.encode_images(query_img)
        feats = ImageFeatures(torch.cat([f.tensor, db_feat.tensor], dim=1), 33, f.generation)
        return [model.decode(model.encode_context_pairs(feats, pairs_a[k:k + BATCH], reuse=True), q)["pred_corrs"]
                for k, q in zip(range(0, 32, BATCH), q_a)]

    # (b) all 56 ordered pairs of 8 images
    imgs_b = rand(8, 3, 256, 256)
    pairs_b = [(i, j) for i in range(8) for j in range(8) if i != j]
    canv_b = [canvases(imgs_b, pairs_b[k:k + BATCH]).contiguous() for k in range(0, 56, BATCH)]
    q_b = [uniform(BATCH, Q, 2) for _ in range(0, 56, BATCH)]

    def canvas_b():
        return [model(c, q)["pred_corrs"] for c, q in zip(canv_b, q_b)]

    def features_b():
        feats = model.encode_images(imgs_b)
        return [model.decode(model.encode_context_pairs(feats, pairs_b[k:k + BATCH], reuse=True), q)["pred_corrs"]
                for k, q in zip(range(0, 56, BATCH), q_b)]

    def one_pair_at_a_time(canv, qs):
        """the canvas forward of every pair alone: how far the canvas path itself moves with the batch composition"""
        return torch.cat([model(c[i:i + 1], q[i:i + 1])["pred_corrs"] for c, q in zip(canv, qs) for i in range(c.shape[0])])

    result = dict(card=card(), torch_device=torch.cuda.get_device_name(), Q=Q, batch_pairs=BATCH, repeats=args.repeats)
    failed = []
    for name, n_pairs, arms, canv, qs in (("a_query_vs_32_db", 32, (canvas_a, features_a), canv_a, q_a),
                                          ("b_all_pairs_of_8", 56, (canvas_b, features_b), canv_b, q_b)):
        for fn in arms:
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        ref, got = torch.cat(arms[0]()), torch.cat(arms[1]())
        single = one_pair_at_a_time(canv, qs)
        diff = (ref - got).abs().max().item()
        drift = (ref - single).abs().max().item()
        times = ([], [])
        for _ in range(args.repeats):
            for t, fn in zip(times, arms):
                t.append(timed(fn)[0])
        ms = [float(np.median(t)) for t in times]
        spread = [(float(np.min(t)), float(np.max(t))) for t in times]
        row = dict(pairs=n_pairs, max_abs_diff=diff, agree=diff < max(AGREE_TOL, 2 * drift), canvas_batch_drift=drift,
                   features_vs_one_pair_canvas=(got - single).abs().max().item(),
                   canvas_ms_per_step=ms[0], features_ms_per_step=ms[1],
                   canvas_ms_per_step_min_max=spread[0], features_ms_per_step_min_max=spread[1],
                   canvas_ms_per_pair=ms[0] / n_pairs, features_ms_per_pair=ms[1] / n_pairs,
                   canvas_qps=n_pairs * Q / (ms[0] * 1e-3), features_qps=n_pairs * Q / (ms[1] * 1e-3),
                   speedup=ms[0] / ms[1])
        result[name] = row
        print(f"{name}: canvas {row['canvas_ms_per_pair']:.3f} ms/pair ({row['canvas_qps'] / 1e6:.2f} M query points/s), "
              f"features {row['features_ms_per_pair']:.3f} ms/pair ({row['features_qps'] / 1e6:.2f} M/s), "
              f"x{row['speedup']:.2f}, max |features - canvas| {diff:.2e} (canvas 8 pairs vs 1 pair per forward: "
              f"{drift:.2e}; features vs 1 pair per forward: {row['features_vs_one_pair_canvas']:.2e})", flush=True)
        if not row["agree"]:
            failed.append(f"{name}: the arms disagree by {diff:.2e}")

    db_ms = [timed(lambda: model.encode_images(db))[0] for _ in range(args.repeats)]
    result["a_database_encode_ms"] = float(np.median(db_ms))
    print(f"one-off database encode (32 images): {result['a_database_encode_ms']:.3f} ms; card: {result['card']}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    assert not failed, "; ".join(failed)


if __name__ == "__main__":
    main()
