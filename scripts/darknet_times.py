"""Throughput of the DarkNet classifier plans, their launch times, and the same networks in PyTorch eager.

    python scripts/darknet_times.py [--batch 256] [--size 224] [--iters 30] [--archs n,s,m,l,x] [--json out.json]

Reports, from CUDA events on the current card (its name and power limit are read in the same run), for each r6.0
classifier at the given batch and square canvas in fp16:
  * the whole plan replayed as a CUDA graph: time and images per second;
  * the time of every launch; the head launches (AVGPOOL, classifier.0, classifier.3) are listed on their own, the
    AVGPOOL one with the bytes it moves (from the shapes) and the achieved rate against the H100 SXM data-sheet HBM3
    bandwidth of 3.35 TB/s;
  * the same network in PyTorch eager, fp16, channels_last (F.conv2d / batch_norm / SiLU / C3 as the reference's
    modules compute them, restated by oracle/restate_darknet.py).
Synthetic weights (oracle/make_golden_darknet.py); nothing is written to the tree."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden_darknet import synth_state_dict_darknet  # noqa: E402
from oracle.restate_darknet import NetDarknet  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.models import darknet as D  # noqa: E402

HBM_BPS = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def time_ms(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--archs", default="n,s,m,l,x")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("darknet_times.py measures on a GPU; none is visible")
    N, H, W = args.batch, args.size, args.size
    name, power = card()
    print(f"card: {name}  power.limit, clocks.max.sm: {power}")
    torch.backends.cudnn.benchmark = True
    results = {}
    for s in args.archs.split(","):
        arch = f"darknet_{s}_r6_0"
        m = getattr(D, arch)().eval()
        sd = synth_state_dict_darknet({k: list(v.shape) for k, v in m.state_dict().items()})
        m.load_state_dict(sd)
        m = m.to("cuda:0", torch.float16)
        plan = m.get_plan(N, H, W)
        g = torch.Generator(device="cuda:0").manual_seed(0)
        plan.input.copy_(torch.rand(plan.input.shape, generator=g, device="cuda:0").half())
        plan.input[..., 3::4] = 0
        L = plan._low.L
        rows = []
        for li, grp in enumerate(plan.launch_ops):
            op = L.ops[grp[0]]
            us = time_ms(lambda: plan.run(li, 1), args.iters) * 1e3
            row = {"launch": plan.op_names[li], "kind": op.kind, "us": us, "flops": plan.op_flops[li]}
            if op.kind == _C.YB_OP_AVGPOOL:
                h, w = op.src.buf.hw(H, W)
                row["bytes"] = N * (h * w + 1) * op.src.C * 2
            rows.append(row)
        head = rows[-3:]
        plan.use_graph = True
        plan_ms = time_ms(plan.run, args.iters)
        # comparator: the same network in PyTorch eager, fp16 channels_last
        net = NetDarknet(sd)
        net.sd = {k: v.to("cuda:0", torch.float16) for k, v in net.sd.items()}
        x = torch.rand(N, 3, H, W, generator=g, device="cuda:0").half().to(memory_format=torch.channels_last)
        with torch.no_grad():
            eager_ms = time_ms(lambda: net.classifier(net.avgpool(net.features(x))), args.iters)
        print(f"\n{arch} N={N} {H}x{W} f16: plan (graph replay) {plan_ms:.3f} ms  {N / plan_ms * 1e3:.0f} img/s;  "
              f"PyTorch eager fp16 channels_last {eager_ms:.3f} ms  {N / eager_ms * 1e3:.0f} img/s;  "
              f"sum of launches {sum(r['us'] for r in rows) / 1e3:.3f} ms ({len(rows)} launches)")
        for r in head:
            extra = ""
            if "bytes" in r:
                bps = r["bytes"] / (r["us"] * 1e-6)
                extra = f"  {r['bytes'] / 1e6:.2f} MB  {bps / 1e9:.0f} GB/s  {100 * bps / HBM_BPS:.1f}% of 3.35 TB/s"
            elif r["flops"]:
                extra = f"  {r['flops'] / 1e9:.2f} GFLOP  {r['flops'] / (r['us'] * 1e-6) / 1e12:.1f} TFLOP/s"
            print(f"  head launch {r['us']:8.1f} us  {r['launch']}{extra}")
        results[arch] = {"plan_ms": plan_ms, "img_s": N / plan_ms * 1e3, "eager_ms": eager_ms,
                         "eager_img_s": N / eager_ms * 1e3, "launches": rows}
        del plan, m, net
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power": power, "N": N, "H": H, "W": W, "archs": results}, f, indent=1)


if __name__ == "__main__":
    main()
