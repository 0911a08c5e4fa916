"""Launch times of the yolov5_mobilenet_v3_small_fpn plan, and the same network in PyTorch eager as a comparator.

    python scripts/lite_times.py [--batch 32] [--size 640] [--iters 50] [--json out.json]

Reports, from CUDA events on the current card (its name and power limit are read in the same run):
  * the time of every launch of the plan, and for each depthwise / squeeze-excitation launch the bytes it has to move
    (from the shapes) and the achieved rate against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s;
  * the whole plan replayed as a CUDA graph: time and images per second;
  * torchvision's MobileNetV3 features + FPN + the 1x1 heads in PyTorch eager, fp16, channels_last, on the same card.
Synthetic weights (oracle/make_golden_lite.py); nothing is written to the tree."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden_lite import synth_state_dict_lite  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.models.yolo_lite import yolov5_mobilenet_v3_small_fpn  # noqa: E402

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


def op_bytes(op, N, H, W):
    """Bytes a depthwise or SE launch must move at least (activations, weights, biases)."""
    hi, wi = H // op.src.buf.div, W // op.src.buf.div
    ho, wo = H // op.dst.buf.div, W // op.dst.buf.div
    C = op.src.C
    wb = op.weight.numel() * op.weight.element_size() + op.bias.numel() * 4
    if op.kind == _C.YB_OP_DWCONV:
        return N * (hi * wi + ho * wo) * C * 2 + wb
    return N * hi * wi * C * 2 * 3 + wb      # SE: read for the mean, read again and write for the scale


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lite_times.py measures on a GPU; none is visible")
    N, H, W = args.batch, args.size, args.size
    name, power = card()
    print(f"card: {name}  power.limit, clocks.max.sm: {power}")

    m = yolov5_mobilenet_v3_small_fpn(pretrained_backbone=False).eval()
    m.load_state_dict(synth_state_dict_lite({k: list(v.shape) for k, v in m.state_dict().items()}))
    m = m.to("cuda:0")
    plan = m.engine().plan(N, H, W)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    plan.input.copy_(torch.rand(plan.input.shape, generator=g, device="cuda:0").half())
    plan.input[..., 3::4] = 0
    L = plan._low.L

    rows = []
    for li, grp in enumerate(plan.launch_ops):
        op = L.ops[grp[0]]
        ms = time_ms(lambda: plan.run(li, 1), args.iters)
        row = {"launch": plan.op_names[li], "kind": op.kind, "us": ms * 1e3}
        if op.kind in (_C.YB_OP_DWCONV, _C.YB_OP_SE):
            nb = op_bytes(op, N, H, W)
            row.update(bytes=nb, GBps=nb / (ms * 1e-3) / 1e9, of_hbm=nb / (ms * 1e-3) / HBM_BPS)
        rows.append(row)
        extra = f"  {row['bytes'] / 1e6:8.2f} MB  {row['GBps']:7.0f} GB/s  {100 * row['of_hbm']:5.1f}% of 3.35 TB/s" \
            if "bytes" in row else ""
        print(f"{li:3d} {row['us']:9.1f} us  {row['launch']}{extra}")
    dw = [r for r in rows if r["kind"] == _C.YB_OP_DWCONV]
    se = [r for r in rows if r["kind"] == _C.YB_OP_SE]
    print(f"sum of launches {sum(r['us'] for r in rows) / 1e3:.3f} ms;  depthwise {sum(r['us'] for r in dw):.0f} us "
          f"({sum(r['bytes'] for r in dw) / 1e6:.0f} MB);  SE {sum(r['us'] for r in se):.0f} us "
          f"({sum(r['bytes'] for r in se) / 1e6:.0f} MB)")

    plan.use_graph = True
    plan_ms = time_ms(plan.run, args.iters)
    print(f"plan (graph replay) N={N} {H}x{W} f16: {plan_ms:.3f} ms  {N / plan_ms * 1e3:.0f} img/s")

    # comparator: torchvision's own modules, PyTorch eager, fp16 channels_last
    body = m.backbone.body.half().to(memory_format=torch.channels_last)
    fpn = m.backbone.fpn.half().to(memory_format=torch.channels_last)
    heads = m.head.head.half().to(memory_format=torch.channels_last)
    x = torch.rand(N, 3, H, W, generator=g, device="cuda:0").half().to(memory_format=torch.channels_last)

    def eager():
        feats = list(fpn(body(x)).values())
        return [h(f) for h, f in zip(heads, feats)]

    with torch.no_grad():
        eager_ms = time_ms(eager, args.iters)
    print(f"PyTorch eager fp16 channels_last N={N} {H}x{W}: {eager_ms:.3f} ms  {N / eager_ms * 1e3:.0f} img/s")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power": power, "N": N, "H": H, "W": W, "launches": rows, "plan_ms": plan_ms,
                       "eager_ms": eager_ms}, f, indent=1)


if __name__ == "__main__":
    main()
