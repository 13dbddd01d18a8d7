"""Check that two builds of the library launch the same kernels and compute the same bits.

    python tools/compare_builds.py OLD.so NEW.so [--out DIR]

Each library runs a fixed matrix of calls in a subprocess of its own (capi.LIB_PATH is set before the first load), on
seeded inputs from cotr_b200.utils.synthetic.  For every call the subprocess dumps the profiler records
(kernel, M, N, K), the launch count and every output; the parent process then requires identical records and launch
counts and byte-identical arrays (so NaNs compare equal).  Records come from eager calls, because the profiler
disables graph replay; the outputs of three more forwards per shape (eager, capture, replay) are compared as well.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FORWARD_TC = [(1, 1024), (2, 100), (4, 1024), (1, 4096)]
VARIANT_SHAPES = [(1, 1024), (2, 100)]
RAGGED_COUNTS = [3, 0, 100, 1500, 40000]


def dump(lib_path, out_prefix):
    sys.path.insert(0, REPO)
    from cotr_b200 import capi
    capi.LIB_PATH = lib_path
    import torch
    from cotr_b200.utils import synthetic

    lib = capi.lib()
    model = capi.NativeModel(synthetic.make_state_dict(0), 0)
    arrays, meta = {}, {}

    def inputs(seed, B, Q):
        img, q = synthetic.make_inputs(seed, B, Q)
        return torch.from_numpy(img).cuda(), torch.from_numpy(q).cuda()

    def profiled(name, fn):
        model.profile_begin(8192)
        outs = fn() or []
        recs = [list(r[:4]) for r in model.profile_end()]
        meta[name] = {"records": recs, "launches": model.last_launch_count()}
        for i, o in enumerate(outs):
            arrays[f"{name}/{i}"] = o.detach().cpu().numpy() if isinstance(o, torch.Tensor) else np.asarray(o)

    def forwards(tag, B, Q, debug=False):
        img, q = inputs(B * 1000 + Q, B, Q)
        profiled(f"{tag}/fwd{B}x{Q}/eager", lambda: [model.forward(img, q)])
        if debug:
            names = {"feat": B * 2 * 256 * 1024, "src": B * 512 * 256, "mem": B * 512 * 256, "hs": B * Q * 256}
            for n, size in names.items():
                arrays[f"{tag}/fwd{B}x{Q}/debug_{n}"] = model.debug_read(n, size)
        for i in range(3):       # first call, capture, replay
            pred = model.forward(img, q)
            torch.cuda.synchronize()
            arrays[f"{tag}/fwd{B}x{Q}/graph{i}"] = pred.cpu().numpy()
            meta[f"{tag}/fwd{B}x{Q}/graph{i}"] = {"records": [], "launches": model.last_launch_count()}

    def set_variant(v):
        lib.cotr_debug_set_variant(v)
        model.set_gemm_path(1)          # a path switch drops the captured graphs, so the new variant is captured
        model.set_gemm_path(0)

    # forward on the tensor-core path, then under the two variant bits that pin the LayerNorm schedules
    for B, Q in FORWARD_TC:
        forwards("tc", B, Q, debug=(B, Q) in [(1, 1024), (4, 1024)])
    for v in (1 << 16, 1 << 19):
        set_variant(v)
        for B, Q in VARIANT_SHAPES:
            forwards(f"variant{v}", B, Q)
    set_variant(0)
    # fp32 SIMT path
    model.set_gemm_path(1)
    forwards("simt", 2, 100)
    model.set_gemm_path(0)

    # cached image features -> pair contexts -> decode
    imgs = torch.from_numpy(synthetic.make_inputs(7, 2, 1)[0]).cuda()          # (2,3,256,512): 4 images of 256x256
    images = torch.cat([imgs[:, :, :, :256], imgs[:, :, :, 256:]]).contiguous()
    ctx = capi.NativeContext(model, 5)
    profiled("features/encode_images", lambda: [model.encode_images(images)])
    feat = model.encode_images(images)
    pairs = np.array([[0, 1], [2, 3], [1, 2]], dtype=np.int32)
    profiled("features/encode_pairs", lambda: model.encode_context_pairs(feat, pairs, ctx))
    _, q = inputs(11, 3, 500)
    profiled("features/decode", lambda: [model.decode(ctx, q)])

    # ragged decode on both paths, over a 5-pair context
    img5, _ = inputs(13, 5, 1)
    offsets = np.concatenate([[0], np.cumsum(RAGGED_COUNTS)]).astype(np.int64)
    qr = torch.rand((int(offsets[-1]), 2), generator=torch.Generator().manual_seed(17)).cuda()
    for path in (0, 1):
        model.set_gemm_path(path)
        profiled(f"ragged{path}/encode", lambda: model.encode_context(img5, ctx))
        profiled(f"ragged{path}/decode", lambda: [model.decode_ragged(ctx, qr, offsets)])
    model.set_gemm_path(0)

    # attention maps
    img2, q2 = inputs(19, 2, 300)
    for path, v in ((0, 0), (0, 1 << 16), (0, 1 << 19), (1, 0)):
        model.set_gemm_path(path)
        lib.cotr_debug_set_variant(v)
        tag = f"maps_path{path}_variant{v}"
        profiled(f"{tag}/encode", lambda: [model.encode_context_attention(img2, ctx, 0b100001)])
        profiled(f"{tag}/decode", lambda: list(model.decode_attention(ctx, q2, 0b010010)))
    lib.cotr_debug_set_variant(0)
    model.set_gemm_path(0)

    torch.cuda.synchronize()
    np.savez(out_prefix + ".npz", **arrays)
    with open(out_prefix + ".json", "w") as f:
        json.dump(meta, f)
    ctx.close()
    model.close()


def compare(old_prefix, new_prefix):
    problems = []
    with open(old_prefix + ".json") as f:
        old_meta = json.load(f)
    with open(new_prefix + ".json") as f:
        new_meta = json.load(f)
    if sorted(old_meta) != sorted(new_meta):
        problems.append("different call lists")
    for k in sorted(set(old_meta) & set(new_meta)):
        if old_meta[k] != new_meta[k]:
            problems.append(f"{k}: records or launch count differ ({old_meta[k]['launches']} vs {new_meta[k]['launches']})")
    old, new = np.load(old_prefix + ".npz"), np.load(new_prefix + ".npz")
    if sorted(old.files) != sorted(new.files):
        problems.append("different output lists")
    for k in sorted(set(old.files) & set(new.files)):
        a, b = old[k], new[k]
        if a.shape != b.shape or a.dtype != b.dtype or a.tobytes() != b.tobytes():
            problems.append(f"{k}: outputs differ")
    n_records = sum(len(v["records"]) for v in new_meta.values())
    return problems, len(new_meta), len(new.files), n_records


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*")
    ap.add_argument("--out", default=None, help="directory for the dumps and summary.json (default: a temporary one)")
    ap.add_argument("--dump", nargs=2, metavar=("LIB", "PREFIX"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump:
        dump(os.path.abspath(args.dump[0]), args.dump[1])
        return 0
    if len(args.libs) != 2:
        ap.error("expects two library paths")
    out = args.out or tempfile.mkdtemp(prefix="compare_builds_")
    os.makedirs(out, exist_ok=True)
    prefixes = []
    for i, lib in enumerate(args.libs):
        prefix = os.path.join(out, f"dump{i}")
        subprocess.run([sys.executable, os.path.abspath(__file__), "--dump", lib, prefix], check=True)
        prefixes.append(prefix)
    problems, n_calls, n_arrays, n_records = compare(*prefixes)
    summary = {"libs": args.libs, "calls": n_calls, "arrays": n_arrays, "records": n_records, "problems": problems,
               "identical": not problems}
    with open(os.path.join(out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary))
    return 1 if problems else 0


if __name__ == "__main__":
    sys.exit(main())
