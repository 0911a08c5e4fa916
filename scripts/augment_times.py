"""Times the training front end on the GPU: a batch of 32 seeded 640x480 uint8 images (COCO's common size) through
default_train_transforms() (csrc/augment.cu) and the training letterbox (YOLOTransform(640, 640) with targets).

Reports CUDA-event times (median of --iters after warm-up) of
  kernels    the augmentation launches alone, on parameters drawn beforehand
  augment    Compose.apply_batch: host draws + descriptor copy + launches
  step       apply_batch + YOLOTransform(images, targets)
  sampler    the device sampler's kernel alone (augment_sample_kernel, from a torch.profiler pass of its own)
  sampled    Compose.apply_batch(..., generator=g): key draw + copies + sampler + read-back + pixel launches
  sampled step  the same + YOLOTransform(images, targets)
with the bytes each moves (source read once per pass that reads it, output written once) and the fraction of the
H100's 3.35 TB/s that is.  For context it times the same torchvision tensor ops the reference runs, on the CPU, image
by image, on the same recipes.  The card's name and power limit are printed in the same run.

    python scripts/augment_times.py [--batch 32] [--iters 20]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from yolort_b200.data import transforms as T  # noqa: E402
from yolort_b200.models.transform import YOLOTransform  # noqa: E402

HBM = 3.35e12


def batch(n, seed):
    g = torch.Generator().manual_seed(seed)
    images = [torch.randint(0, 256, (3, 480, 640), dtype=torch.uint8, generator=g) for _ in range(n)]
    targets = []
    for _ in range(n):
        k = int(torch.randint(1, 8, (1,), generator=g))
        xy = torch.rand(k, 2, generator=g) * torch.tensor([500.0, 360.0])
        wh = torch.rand(k, 2, generator=g) * torch.tensor([140.0, 120.0]) + 4
        targets.append({"boxes": torch.cat([xy, xy + wh], 1), "labels": torch.randint(0, 80, (k,), generator=g)})
    return images, targets


def aug_bytes(images, states):
    total = 0
    for im, st in zip(images, states):
        src = im.numel()
        rounds = sum(1 for op in st.ops if op[0] == 2)
        total += src * (1 + rounds) + 3 * st.h * st.w * (4 if st.float_out else 1)
    return total


def cpu_apply(im, recipe):
    import torchvision.transforms._functional_tensor as TF

    for op in recipe:
        k = op[0]
        if k == "brightness":
            im = TF.adjust_brightness(im, op[1])
        elif k == "contrast":
            im = TF.adjust_contrast(im, op[1])
        elif k == "saturation":
            im = TF.adjust_saturation(im, op[1])
        elif k == "hue":
            im = TF.adjust_hue(im, op[1])
        elif k == "permute":
            im = im[list(op[1])]
        elif k == "zoom":
            _, ch, cw, top, left, fill = op
            out = torch.empty((3, ch, cw), dtype=torch.uint8)
            out[:] = torch.tensor(fill, dtype=torch.uint8).view(3, 1, 1)
            out[:, top:top + im.shape[1], left:left + im.shape[2]] = im
            im = out
        elif k == "crop":
            im = TF.crop(im, *op[1:])
        elif k == "hflip":
            im = TF.hflip(im)
        elif k == "float":
            im = TF.convert_image_dtype(im, torch.float)
    return im


def events(fn, iters):
    times = []
    for i in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn(i)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def sampler_kernel_us(fn, iters):
    """Median device time of augment_sample_kernel over `iters` calls of `fn`, from a profiler pass of its own."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(iters):
            fn(i)
        torch.cuda.synchronize()
    times = [e.time_range.elapsed_us() for e in prof.events() if "augment_sample_kernel" in e.name]
    if not times:
        raise SystemExit("the profiler recorded no augment_sample_kernel launch")
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-iters", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("augment_times.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {torch.cuda.get_device_name(dev)} | nvidia-smi: {q}")
    host_images, targets = batch(args.batch, 0)
    images = [im.to(dev) for im in host_images]
    pipe = T.default_train_transforms()
    lb = YOLOTransform(640, 640)
    seeds = list(range(args.warmup + args.iters))
    plans = []
    for s in seeds:
        torch.manual_seed(s)
        plans.append(pipe.plan([(480, 640)] * args.batch, [dict(t) for t in targets]))

    def kernels(i):
        T.run_recipes(images, plans[(i + args.warmup) % len(plans)])

    def augment(i):
        torch.manual_seed(i)
        pipe.apply_batch(images, targets)

    def step(i):
        torch.manual_seed(i)
        outs, tg = pipe.apply_batch(images, targets)
        lb(outs, tg)

    g = torch.Generator(dev)

    def sampled(i):
        g.manual_seed(i)
        pipe.apply_batch(images, targets, generator=g)

    def sampled_step(i):
        g.manual_seed(i)
        outs, tg = pipe.apply_batch(images, targets, generator=g)
        lb(outs, tg)

    results = {}
    for name, fn in (("kernels", kernels), ("augment", augment), ("step", step), ("sampled", sampled),
                     ("sampled step", sampled_step)):
        for i in range(args.warmup):
            fn(i)
        torch.cuda.synchronize()
        results[name] = events(fn, args.iters)
    nbytes = statistics.median(aug_bytes(images, p) for p in plans)
    out_px = statistics.median(sum(st.h * st.w for st in p) for p in plans)
    lb_bytes = nbytes + 4 * 3 * out_px + args.batch * 3 * 640 * 640 * 4
    print(f"batch {args.batch} x 480x640 uint8, median of {args.iters} (CUDA events)")
    print(f"  kernels  {results['kernels']:.3f} ms  {nbytes / 1e6:.1f} MB  "
          f"{nbytes / (results['kernels'] * 1e-3) / 1e9:.0f} GB/s = {nbytes / (results['kernels'] * 1e-3) / HBM:.1%} of HBM")
    print(f"  augment  {results['augment']:.3f} ms (host draws + copy + launches)")
    print(f"  step     {results['step']:.3f} ms  {lb_bytes / 1e6:.1f} MB with the letterbox")
    print(f"  sampler  {sampler_kernel_us(sampled, args.iters):.1f} us (augment_sample_kernel alone, median)")
    print(f"  sampled  {results['sampled']:.3f} ms (device sampler + read-back + launches)")
    print(f"  sampled step  {results['sampled step']:.3f} ms")
    torch.set_num_threads(os.cpu_count() or 1)
    t0 = time.perf_counter()
    for it in range(args.cpu_iters):
        for im, st in zip(host_images, plans[it]):
            cpu_apply(im, T.recipe_of(st))
    cpu_ms = (time.perf_counter() - t0) / args.cpu_iters * 1e3
    print(f"  torchvision tensor ops on the CPU ({torch.get_num_threads()} threads, {os.cpu_count()} cores): "
          f"{cpu_ms:.1f} ms per batch")


if __name__ == "__main__":
    main()
