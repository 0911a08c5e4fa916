"""Per-launch CUDA-event times of one plan next to what the launch has to move and compute.

    python scripts/launch_times.py [model] [batch] [size] [reps] [dtype]      (default yolov5s 32 640 20 f16)

For every launch: the median time over `reps` full-plan passes (an event pair around every launch, so each launch sees
the cache state of a real step), the algorithmic bytes (every input, output, residual and weight tensor once, from
the descriptor's shapes), the FLOP, the least time the data-sheet H100 SXM could take (the larger of bytes / 3.35 TB/s
and FLOP / 989 TFLOP/s dense FP16), which of the two bounds it, and the layout the launch was planned for
(yb_conv_config): CTAs per SM x consumer warpgroups per CTA, 1x2, 2x2 (the 104-register instances) or 2x1, and the
rounds of the persistent grid (work items / grid; "+s" when the tiles of a partial last round run as s column slices).
The card's name and power limit are printed with the table."""
import ctypes
import subprocess
import sys

sys.path.insert(0, ".")
import torch

import yolort_b200.models as M
from yolort_b200 import _C

HBM_BPS = 3.35e12
FP16_FLOPS = 989e12

name = sys.argv[1] if len(sys.argv) > 1 else "yolov5s"
batch = int(sys.argv[2]) if len(sys.argv) > 2 else 32
size = int(sys.argv[3]) if len(sys.argv) > 3 else 640
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 20
dt = sys.argv[5] if len(sys.argv) > 5 else "f16"
dev = torch.device("cuda:0")


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "nvidia-smi unavailable"


def launch_bytes(d) -> int:
    """Bytes a launch must read and write at least once (2-byte activations and weights)."""
    esz = 2
    px_in, px_out = d.N * d.H * d.W, d.N * d.Ho * d.Wo
    b = px_in * d.Cin * esz
    if d.kind == _C.YB_OP_CONV:
        b += d.Cout_pad * d.ksize * d.ksize * d.Cin_pad * esz
        if d.residual:
            b += px_out * d.Cout * esz
        if d.chain:
            c = _C.ConvChain.from_address(d.chain)
            b += c.Cout_pad * c.K_pad * esz + px_out * c.Cout * esz
            if c.extra:
                b += px_out * c.extra_C * esz
            if c.store_first:
                b += px_out * d.Cout * esz
        else:
            b += px_out * d.Cout * esz
    else:
        b += px_out * d.Cout * esz
    return b


torch.manual_seed(0)
m = getattr(M, name)(score_thresh=0.25, size=(size, size)).eval().to(dev)
if dt == "bf16":
    m = m.to(torch.bfloat16)
plan = m.model.get_plan(batch, size, size)
n = plan.plan.n_ops
descs = plan._descs
for _ in range(20):
    plan.run()
torch.cuda.synchronize()
ev = [[torch.cuda.Event(enable_timing=True) for _ in range(n + 1)] for _ in range(reps)]
for r in range(reps):
    ev[r][0].record()
    for i in range(n):
        plan.run(i, 1)
        ev[r][i + 1].record()
torch.cuda.synchronize()

print(f"# {name} batch {batch} {size}x{size} {dt} on {card()}")
print(f"# per-launch us: median of {reps} full-plan passes; bound = max(bytes / 3.35 TB/s, FLOP / 989 TFLOP/s)")
print(f"{'op':>3} {'us':>8} {'MB':>8} {'GFLOP':>7} {'bound us':>8} {'by':>4} {'of bound':>8} {'layout':>6} {'rounds':>7}  launch")
tot = tot_bound = 0.0
for i in range(n):
    ts = sorted(ev[r][i].elapsed_time(ev[r][i + 1]) * 1e3 for r in range(reps))
    t = ts[len(ts) // 2]
    d = descs[i]
    by = launch_bytes(d)
    fl = plan.op_flops[i]
    t_mem, t_mma = by / HBM_BPS * 1e6, fl / FP16_FLOPS * 1e6
    bound = max(t_mem, t_mma)
    layout = rounds = "-"
    if d.kind == _C.YB_OP_CONV:
        cfg = _C.conv_config(d)
        layout = cfg["layout"]
        rounds = f"{cfg['work_items'] / cfg['grid']:.2f}" + (f"+{cfg['tail_split']}" if cfg["tail_split"] > 1 else "")
    tot += t
    tot_bound += bound
    print(f"{i:3d} {t:8.1f} {by / 1e6:8.1f} {fl / 1e9:7.2f} {bound:8.1f} {'HBM' if t_mem >= t_mma else 'MMA':>4} "
          f"{bound / t:8.2f} {layout:>6} {rounds:>7}  {plan.op_names[i]}")
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(reps):
    plan.run()
e1.record()
torch.cuda.synchronize()
print(f"# sum of launches {tot:.1f} us (bound {tot_bound:.1f} us); plan back-to-back {e0.elapsed_time(e1) / reps * 1e3:.1f} us; "
      f"GFLOP {sum(plan.op_flops) / 1e9:.1f}")
