"""Per-launch profile of the backbone GEMMs of one forward (default B=1, Q=1024), eager, L2 flushed before each pass.

For each of the 43 backbone launches (stem, then conv1 / conv2 / downsample / conv3 of every bottleneck) prints M, N, K,
the median time over the passes (library profiler: CUDA events around each launch) and the achieved operand rate:
the bytes every CTA stages from L2 into shared memory, summed over the launch, over that time.  The byte model follows
the tile rules of csrc/gemm_tc.cu (launch_gemm_tc / launch_one): a CTA of a 128 x BN tile stages BN x K' weight
halves and either 128 x K' activation halves (implicit im2col: every 3x3 tap of a pixel is copied again) or, for the
halo loader of the stride-1 3x3 convolutions, each 64-channel halo tile once; two fp16 planes each.

    python tools/backbone_profile.py [--B 1] [--Q 1024] [--passes 10] [--variant 0] [--json out.json]
"""
import argparse
import json
import math
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

WAVE_CTAS = 144          # gemm_tc.cu kWaveCtas
NUM_SMS = 132            # common.cuh kNumSms: the wave limit of the halo loader's split-K
HALO_MAX_BYTES = 100 * 1024   # gemm_tc.cu kHaloMaxBytes
HALO_MIN_CTAS = 86            # gemm_tc.cu kHaloMinCtas


def backbone_convs():
    """(name, cin, cout, k, stride, H_in) in launch order: the stem, then torchvision Bottleneck blocks to layer3."""
    convs = [("stem", 3, 64, 7, 2, 256)]
    cin, H = 64, 64
    for li, (planes, blocks, stride) in enumerate([(64, 3, 1), (128, 4, 2), (256, 6, 2)], start=1):
        for b in range(blocks):
            s = stride if b == 0 else 1
            p = f"layer{li}.{b}"
            convs.append((p + ".conv1", cin, planes, 1, 1, H))
            convs.append((p + ".conv2", planes, planes, 3, s, H))
            if b == 0:
                convs.append((p + ".downsample", cin, planes * 4, 1, s, H))
            convs.append((p + ".conv3", planes, planes * 4, 1, 1, H // s))
            cin = planes * 4
            H //= s
    return convs


def halo_geometry(n_img, H, W, C):
    """Row tiles, per-chunk halo rows and bytes of the halo loader (gemm_tc.cu LD_HALO) for a 3x3 stride-1 conv."""
    tiles_per_img = math.ceil(H * (W + 2) / 128)
    rows = 128 + 2 * (W + 2) + 2
    chunk_bytes = 2 * ((rows + 7) // 8 * 8) * 128
    return n_img * tiles_per_img, rows, chunk_bytes


def launch_bytes(name, M, N, K, n_img, H_in, stride, k, variant, halo):
    """(CTAs, operand bytes staged from L2 into shared memory by the whole launch)."""
    C = K // (k * k) if name != "stem" else 0
    use_halo = halo and k == 3 and stride == 1 and not (variant & (1 << 20))
    if use_halo:
        mt, rows, chunk_bytes = halo_geometry(n_img, H_in, H_in, C)
    else:
        mt = math.ceil(M / 128)
    thr = [86, 43, 57, 132][(variant >> 10) & 3]
    bn = 64 if (mt * math.ceil(N / 64) >= thr or name == "stem" or N % 32) else 32
    ctas = mt * math.ceil(N / bn)
    kc = math.ceil(K / 64)
    ksplit = 1
    if name != "stem" and bn <= 64 and not (variant & 512) and kc >= (16 >> ((variant >> 14) & 3)):
        cc = C // 64 if use_halo else kc
        wave = NUM_SMS if use_halo else WAVE_CTAS
        if kc % 4 == 0 and cc % 4 == 0 and ctas * 4 <= wave:
            ksplit = 4
        elif kc % 2 == 0 and cc % 2 == 0 and ctas * 2 <= wave:
            ksplit = 2
    if use_halo and ((C // 64 // ksplit) * chunk_bytes > HALO_MAX_BYTES or ctas * ksplit < HALO_MIN_CTAS):
        return launch_bytes(name, M, N, K, n_img, H_in, stride, k, variant, False)    # implicit im2col (launch_one)
    ctas *= ksplit
    w_bytes = ctas * bn * (kc // ksplit) * 64 * 4
    if use_halo:
        a_bytes = ctas * (C // 64 // ksplit) * rows * 128 * 2
    else:
        a_bytes = ctas * 128 * (kc // ksplit) * 64 * 4
    return ctas, a_bytes + w_bytes, use_halo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=1)
    ap.add_argument("--Q", type=int, default=1024)
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--variant", type=int, default=0)
    ap.add_argument("--im2col-only", action="store_true", help="byte model of a build without the halo loader")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from cotr_b200 import capi
    from cotr_b200.models import build_model
    from cotr_b200.utils import synthetic as fixtures

    sd = fixtures.make_state_dict(0)
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    model = model.cuda().eval()
    nat = model.native()
    capi.lib().cotr_debug_set_variant(args.variant)
    nat.set_graph_mode(False)
    img, q = fixtures.make_inputs(1, args.B, args.Q)
    img = torch.from_numpy(img).cuda()
    q = torch.from_numpy(q).cuda()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        model(img, q)
    torch.cuda.synchronize()
    passes = []
    for _ in range(args.passes):
        flush.zero_()
        torch.cuda.synchronize()
        nat.profile_begin()
        model(img, q)
        passes.append(nat.profile_end())
    capi.lib().cotr_debug_set_variant(0)

    convs = backbone_convs()
    gemm_idx = [i for i, r in enumerate(passes[0]) if r[0] == "gemm_tc"][: len(convs)]
    n_img = 2 * args.B
    rows = []
    total_ms = 0.0
    for j, (name, cin, cout, k, stride, H_in) in enumerate(convs):
        i = gemm_idx[j]
        _, M, N, K, _ = passes[0][i]
        ms = float(np.median([p[i][4] for p in passes]))
        ctas, nbytes, halo = launch_bytes(name, M, N, K, n_img, H_in, stride, k, args.variant, not args.im2col_only)
        total_ms += ms
        rows.append(dict(name=name, M=M, N=N, K=K, ctas=ctas, halo=halo, ms=ms, operand_MB=nbytes / 1e6,
                         operand_TBps=nbytes / (ms * 1e-3) / 1e12))
        print(f"{name:22s} M {M:6d} N {N:5d} K {K:5d}  CTAs {ctas:4d} {'halo' if halo else '    '}  "
              f"{ms * 1e3:7.2f} us  {nbytes / 1e6:7.1f} MB  {nbytes / (ms * 1e-3) / 1e12:5.2f} TB/s", flush=True)
    all_ms = sum(float(np.median([p[i][4] for p in passes])) for i in range(len(passes[0])))
    print(f"backbone GEMMs: {total_ms:.3f} ms of {all_ms:.3f} ms summed eager kernel time ({len(passes[0])} launches)")
    stride1 = [r for r in rows if r["name"].endswith("conv2") and r["name"] not in ("layer2.0.conv2", "layer3.0.conv2")]
    print(f"stride-1 3x3 convolutions ({len(stride1)}): {sum(r['ms'] for r in stride1):.3f} ms")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(dict(B=args.B, Q=args.Q, variant=args.variant, gpu=torch.cuda.get_device_name(),
                           launches=rows, backbone_ms=total_ms, all_ms=all_ms), f, indent=1)


if __name__ == "__main__":
    main()
