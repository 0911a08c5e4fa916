#!/usr/bin/env python
"""Headline benchmark: images/sec end-to-end (letterbox -> NMS), yolov5s, batch 32, 640x640, fp16.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config c2|c3|c4|c5] [--scaling weak|strong]
                    [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 ... bench.py --gpus N ...

`--config` selects one of BASELINE.json's configs (default c2 = configs[1], the headline):
    c2  yolov5s batch 32 640x640 fp16            c3  yolov5m batch 128 640x640 bf16 (global batch sharded over the GPUs)
    c4  yolov5l batch 16, mixed 416-1280 sizes, 24 distinct canvases, fp16      c5  yolov5x batch 64 1280x1280 fp16
`--scaling strong` keeps the GLOBAL batch fixed as N grows (c2: 32/N images per GPU); c3 is always strong.

One "step" = one pass of the whole hot path over one batch of 32 synthetic uint8 640x640 images per GPU
(weak scaling: every rank processes its own batch; weights replicated; for N > 1 the padded detections of all
ranks are all-gathered over NCCL inside the step so rank 0 holds a single output list).

Prints ONE JSON line (rank 0).  `value` = whole-job images/s with the uint8 inputs already resident in HBM
(CUDA events around exactly K steps, barrier + synchronize on both sides, max over ranks); `e2e` = same
metric through the public API (`model.predict`) from pinned HOST tensors with the H2D copies and the D2H of the
results inside the timed region.  `roofline` is the tensor-core roofline of the convolution launches (live CUDA
events around the plan); `cpu_baseline` is the CPU oracle port of the reference path on this box's host cores.

`--dump-outputs DIR` writes what the timed path returned in its last timed step (rank 0): the padded detections
boxes [n, D, 4], scores [n, D], labels [n, D] (slots past an image's count zeroed) and the per-image counts [n], as
float32 .npy files.  Inputs and weights
are seeded, so two builds run with the same arguments can be compared output for output.

`--impl reference` times the reference algorithm's CPU port (oracle/restate.py: the reference's own PyTorch CPU
operators in fp32) with every host thread, on a bounded sample of the same workload per step.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

BATCH = 32
SIZE = 640
MODEL = "yolov5s"
SCORE_THRESH = 0.25
# BASELINE.json configs[1..4]: model, global/per-GPU batch, canvas, dtype, how the batch relates to the GPU count
CONFIGS = {
    # `thr`: score threshold giving ~1000-1500 candidates per image with the config's weights (calibrated on the oracle)
    "c2": dict(model="yolov5s", batch=32, size=640, dtype="f16", scaling="weak", gain=None, thr=0.25,
               what="yolov5s batch 32/GPU 640x640 uint8 -> detections (configs[1])"),
    "c3": dict(model="yolov5m", batch=128, size=640, dtype="bf16", scaling="strong", gain=1.4, thr=0.18,
               what="yolov5m GLOBAL batch 128 640x640 uint8 bf16, sharded over the GPUs (configs[2])"),
    "c4": dict(model="yolov5l", batch=16, size=640, dtype="f16", scaling="weak", gain=1.4, mixed=True, thr=0.095,
               what="yolov5l batch 16/GPU, image sizes drawn from 416..1280 (incl. 800/950/523), 24 distinct canvases (configs[3])"),
    "c5": dict(model="yolov5x", batch=64, size=1280, dtype="f16", scaling="weak", gain=1.3, thr=0.044,
               what="yolov5x batch 64/GPU 1280x1280 uint8 -> detections (configs[4])"),
}
GFLOP_PER_IMAGE = {"yolov5n": 4.468, "yolov5s": 16.434, "yolov5m": 48.872, "yolov5l": 108.994, "yolov5x": 205.448}
CPU_SAMPLE_IMAGES = 8          # images per CPU step (bounded sample of the bs32 workload)


def make_state_dict(model, seed: int = 0):
    """Random-init weights of the named architecture (no checkpoints offline): conv ~ N(0, 2/fan_in), BN
    statistics randomised (so folding is exercised), head weights/biases scaled ("load knob") so that about a
    thousand candidates per image pass score_thresh=0.25 and the NMS does real work (300 detections/image).  Pure function of (key, shape)."""
    import zlib

    sd = {}
    for k, v in model.state_dict().items():
        g = torch.Generator().manual_seed((zlib.crc32(k.encode()) + 7919 * seed) & 0x7FFFFFFF)
        shp = tuple(v.shape)
        if k.endswith("num_batches_tracked"):
            t = torch.zeros(shp, dtype=torch.int64)
        elif k.endswith(".weight") and len(shp) == 4:
            t = torch.randn(shp, generator=g) * (2.0 / (shp[1] * shp[2] * shp[3])) ** 0.5
            if ".head.head." in k:
                t = t * 10.0   # spread the logits (random images give nearly constant features)
        elif k.endswith("bn.weight") or k.endswith("running_var"):
            t = torch.rand(shp, generator=g) + 0.5
        elif k.endswith("bn.bias") or k.endswith("running_mean"):
            t = torch.randn(shp, generator=g) * 0.1
        else:  # head bias [3*(nc+5)]
            b = torch.randn(shp, generator=g).view(3, -1) * 0.1
            b[:, 4] += -3.0
            b[:, 5:] += -4.5
            t = b.reshape(-1)
        sd[k] = t
    return sd


def make_images(n: int, seed0: int, size: int = SIZE):
    ims = []
    for i in range(n):
        g = torch.Generator().manual_seed(seed0 + i)
        ims.append(torch.randint(0, 256, (3, size, size), generator=g, dtype=torch.uint8))
    return ims


def make_mixed_images(n: int, seed0: int):
    """configs[3]: H, W ~ randint(416, 1281) (seeded); every batch carries one of the 639-trap sizes 800 / 950 / 523."""
    g = torch.Generator().manual_seed(seed0)
    ims = []
    for i in range(n):
        h, w = (int(v) for v in torch.randint(416, 1281, (2,), generator=g))
        if i == 0:
            h, w = ((800, 600), (950, 523), (523, 950))[seed0 % 3]
        ims.append(torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8))
    return ims


def zoo_state_dict(model, gain: float, seed: int = 1, head_scale: float = 10.0):
    """Weights for m / l / x: conv ~ N(0, gain/fan_in) with He gain < 2 (keeps the deep residual stacks inside fp16
    range, as trained weights do; tests/test_gpu_zoo.py), and the same head "load knob" as make_state_dict: head
    weights x10 (spreads the logits), biases N(0, 0.1) + (-3.0 objectness, -4.5 classes).  With the per-config
    score_thresh of CONFIGS about a thousand candidates per image reach the NMS."""
    import zlib

    from oracle.make_golden import synth_state_dict

    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    sd = synth_state_dict(shapes, knob_obj=0.0, knob_cls=0.0, seed=seed, gain=gain)
    for k in list(sd):
        if ".head.head." in k and k.endswith(".weight"):
            sd[k] = sd[k] * head_scale
        elif ".head.head." in k and k.endswith(".bias"):
            g = torch.Generator().manual_seed(zlib.crc32(k.encode()) & 0x7FFFFFFF)
            b = torch.randn(sd[k].shape, generator=g).view(3, -1) * 0.1
            b[:, 4] += -3.0
            b[:, 5:] += -4.5
            sd[k] = b.reshape(-1)
    return sd


class NvmlClockSampler:
    """SM clock / throttle reasons from NVML, polled by a thread while the timed region runs.  In-process (no
    nvidia-smi start-up inside the timed region: spawning it there shows up as multi-millisecond hiccups in
    individual steps)."""

    def __init__(self, index: int):
        import pynvml

        self.nv = pynvml
        pynvml.nvmlInit()
        # LOCAL_RANK indexes the visible devices; honour CUDA_VISIBLE_DEVICES when it lists plain indices
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "")
        ids = [v for v in vis.split(",") if v.strip().isdigit()]
        phys = int(ids[index]) if index < len(ids) else index
        self.h = pynvml.nvmlDeviceGetHandleByIndex(phys)
        self.mx = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
        self.sm, self.bits, self.stop_flag, self.t = [], 0, False, None

    def _poll(self):
        nv = self.nv
        while not self.stop_flag:
            try:
                self.sm.append(float(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM)))
                self.bits |= int(nv.nvmlDeviceGetCurrentClocksEventReasons(self.h))
            except Exception:
                pass
            time.sleep(0.002)

    def start(self):
        self.t = threading.Thread(target=self._poll, daemon=True)
        self.t.start()

    def stop(self):
        self.stop_flag = True
        if self.t is not None:
            self.t.join(timeout=1)
        nv = self.nv
        names = (("hw_slowdown", nv.nvmlClocksEventReasonHwSlowdown), ("hw_thermal_slowdown", nv.nvmlClocksEventReasonHwThermalSlowdown),
                 ("sw_thermal_slowdown", nv.nvmlClocksEventReasonSwThermalSlowdown), ("sw_power_cap", nv.nvmlClocksEventReasonSwPowerCap))
        sm = sorted(self.sm)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": self.mx,
                "reasons": [n for n, b in names if self.bits & b], "samples": len(sm), "source": "nvml"}


def make_clock_sampler(index: int):
    try:
        return NvmlClockSampler(index)
    except Exception:
        return ClockSampler(index)     # nvidia-smi -lms fallback


class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons while the timed region runs (fallback when NVML is unusable)."""

    QS = (("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
           "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"),
          ("clocks.sm,clocks.max.sm,power.draw,clocks_throttle_reasons.hw_slowdown,clocks_throttle_reasons.hw_thermal_slowdown,"
           "clocks_throttle_reasons.sw_thermal_slowdown,clocks_throttle_reasons.sw_power_cap"))

    def __init__(self, index: int):
        self.index, self.proc, self.lines = index, None, []

    def start(self):
        try:
            q = self.QS[0]
            for cand in self.QS:   # field names differ between driver generations
                probe = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={cand}", "--format=csv,noheader,nounits"],
                                       capture_output=True, text=True, timeout=20)
                if probe.returncode == 0 and len(probe.stdout.strip().split(",")) >= 7:
                    q = cand
                    break
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={q}", "--format=csv,noheader,nounits",
                                          "-lms", "20"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._pump, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                mx = float(f[1])
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


def measured_peaks(sm_mhz=None, sm_max_mhz=None):
    """(tensor TFLOP/s, HBM GB/s, source).  MEASURED_PEAKS.json, when present, holds a burst figure (a kernel timed
    alone, clocks at maximum) and a sustained one (seconds-long loop under the card's power cap): the burst figure is
    the honest denominator when this run's SM clock sat at (>= 95 % of) its maximum, the sustained one otherwise.
    Without it the denominators are NVIDIA's H100 SXM data-sheet figures (dense FP16 989 TFLOP/s, HBM3 3.35 TB/s, at
    up to 700 W), which a power-limited card does not reach."""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    burst = sm_mhz is not None and sm_max_mhz and sm_mhz >= 0.95 * sm_max_mhz
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        key = "bf16_tflops" if burst else "bf16_tflops_sustained"
        return float(d[key]), float(d["hbm_gbs"]), f"measured (MEASURED_PEAKS.json {key}, hbm_gbs)"
    return 989.0, 3350.0, "H100 SXM data sheet (dense FP16, HBM3)"


def cpu_port_images_per_s(sd, steps: int, warmup: int, ims=None, size=(640, 640), thr=SCORE_THRESH):
    """The reference path restated with the reference's own CPU operators (oracle/restate.py), all host threads.
    Returns (images/s, per-step times, detections of the last step)."""
    from oracle import restate as R

    if ims is None:
        ims = make_images(CPU_SAMPLE_IMAGES, 1234)
    # "all the host threads it can use": pick the fastest thread count (oversubscribing a many-core host
    # makes oneDNN/OpenMP convolutions of an 8-image batch much slower than using a few dozen threads)
    ncpu = os.cpu_count() or 1
    best, best_t = ncpu, None
    for nt in sorted({ncpu, min(ncpu, 64), min(ncpu, 32), min(ncpu, 16)}, reverse=True):
        torch.set_num_threads(nt)
        R.detect(sd, ims[:2], score_thresh=thr, size=size)
        t0 = time.perf_counter()
        R.detect(sd, ims[:2], score_thresh=thr, size=size)
        dt = time.perf_counter() - t0
        if best_t is None or dt < best_t:
            best, best_t = nt, dt
    torch.set_num_threads(best)
    times, dets = [], None
    for i in range(warmup + steps):
        t0 = time.perf_counter()
        dets = R.detect(sd, ims, score_thresh=thr, size=size)
        if i >= warmup:
            times.append(time.perf_counter() - t0)
    total = sum(times)
    return len(ims) * len(times) / total, times, dets


def build_model(cfg):
    """(model on the CPU, state dict) of a config: the architecture BASELINE.json names, random-init weights."""
    import yolort_b200.models as M

    ctor = getattr(M, cfg["model"])
    model = ctor(score_thresh=cfg["thr"], size=(cfg["size"], cfg["size"])).eval()
    sd = make_state_dict(model) if cfg["gain"] is None else zoo_state_dict(model, cfg["gain"])
    model.load_state_dict(sd)
    return model, sd


def run_reference(args, rank, world):
    if rank != 0:
        return
    cfg = CONFIGS[args.config]
    model, sd = build_model(cfg)
    n_sample = CPU_SAMPLE_IMAGES if cfg["size"] <= 640 else 1
    ims = make_mixed_images(n_sample, 4321) if cfg.get("mixed") else make_images(n_sample, 1234, cfg["size"])
    ips, times, _ = cpu_port_images_per_s(sd, args.steps, args.warmup, ims, size=(cfg["size"], cfg["size"]), thr=cfg["thr"])
    ms = 1e3 * sum(times) / len(times)
    cores = torch.get_num_threads()
    sample = (f"{n_sample} of the {cfg['batch']} images per step ({args.steps} steps after {args.warmup} warm-up), fp32, "
              f"{cores} threads")
    line = {
        "impl": "reference", "metric": "images/sec end-to-end (letterbox->NMS)", "value": ips, "unit": "images/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True,
        "scaling": cfg["scaling"], "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"{cfg['what']}, score_thresh {cfg['thr']}", "sample": sample},
        "cpu_baseline": {"value": ips, "unit": "images/s", "cores": cores, "kind": "port", "sample": sample},
        "e2e": {"value": ips, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2] if xs else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--precondition", type=int, default=150,
                    help="untimed steps before the warm-up (clock ramp on a cold box); 0 under a profiler")
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="c2", choices=sorted(CONFIGS))
    ap.add_argument("--scaling", default=None, choices=["weak", "strong"],
                    help="weak: the config's batch per GPU; strong: the config's batch in total, split over the GPUs")
    ap.add_argument("--score-thresh", type=float, default=None, help="override the post-process score threshold")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true", help="device-resident leg only (profiling runs)")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the last timed step's detections (boxes, scores, labels, counts) to DIR as float32 .npy")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3)

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        run_reference(args, rank, world)
        return

    import torch.distributed as dist

    cfg = dict(CONFIGS[args.config])
    scaling = args.scaling or cfg["scaling"]
    if scaling == "strong":
        if cfg["batch"] % world:
            raise SystemExit(f"strong scaling: global batch {cfg['batch']} is not divisible by {world} GPUs")
        n_local = cfg["batch"] // world
    else:
        n_local = cfg["batch"]
    size, thr = cfg["size"], (args.score_thresh if args.score_thresh is not None else cfg["thr"])
    if cfg["size"] > 640 and args.precondition > 20:
        args.precondition = 20          # a yolov5x 1280x1280 step is tens of milliseconds: the clocks ramp within a few

    dev = torch.device(f"cuda:{local_rank}")
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    model, sd = build_model(cfg)
    model.model.post_process.score_thresh = thr
    model = model.to(dev)
    if cfg["dtype"] == "bf16":
        model = model.to(torch.bfloat16)

    # inputs: NBUF distinct batches, more than the 50 MB L2 in total, so no step finds its input in L2
    mixed = bool(cfg.get("mixed"))
    per_batch_bytes = n_local * 3 * size * size
    NBUF = 24 if mixed else max(2, min(4, -(-160_000_000 // per_batch_bytes)))
    if mixed:
        host_lists = [[im.pin_memory() for im in make_mixed_images(n_local, 4321 + 7 * b + 1000 * rank)] for b in range(NBUF)]
        dev_lists = [[im.to(dev) for im in hl] for hl in host_lists]
    else:
        host_batches = [torch.stack(make_images(n_local, 1234 + 1000 * b + 100000 * rank, size)).pin_memory() for b in range(NBUF)]
        host_lists = [[hb[j] for j in range(n_local)] for hb in host_batches]
        dev_batches = [hb.to(dev) for hb in host_batches]
        dev_lists = [[db[j] for j in range(n_local)] for db in dev_batches]
    h2d_bytes = int(sum(sum(im.numel() for im in hl) for hl in host_lists) / NBUF)
    D = model.model.post_process.detections_per_img

    gather = None
    if world > 1:
        from yolort_b200.parallel import DetectionGather

        gather = DetectionGather(dev)
    comm_stream = gather.stream if gather is not None else None
    gather_ring = [None, None]

    def step_device(i):
        if gather is not None:
            gather.before_step()
        out = model.forward_padded(dev_lists[i % NBUF])
        if gather is not None:
            # pack + ONE all-gather of the padded detections (the counts ride in an extra row), both on a side stream:
            # they overlap the next step's letterbox / convolutions; the end of the timed region waits for the last one.
            gather_ring[i & 1] = gather.launch(out)          # what a consumer on rank 0 would read: [world, n, D+1, 6]
        return out

    def sync_all():
        torch.cuda.synchronize(dev)     # all streams of the device, the communication stream included
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize(dev)

    # ---- device-resident leg ------------------------------------------------------------------------
    # Untimed preconditioning before the W warm-up steps: a fresh box idles at ~120 MHz and the first launches also
    # pay module loading; W=3..5 steps are ~10 ms, less than the clock ramp.  A fixed count (not a time) so that every
    # rank issues the same collectives.  It also creates the plan of every canvas the timed region will meet.
    for i in range(max(args.precondition, NBUF)):
        step_device(i)
    sync_all()
    for i in range(args.warmup):
        out = step_device(i)
    sync_all()
    engine = model.model.engine()
    n_canvases = len(engine._plans)
    sampler = make_clock_sampler(local_rank)
    if rank == 0:
        sampler.start()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    sync_all()
    ev[0].record()
    for i in range(args.steps):
        out = step_device(i)
        ev[i + 1].record()
    ev_end = torch.cuda.Event(enable_timing=True)
    if world > 1:    # the timed region ends when the LAST gather has landed, not when the last NMS has
        torch.cuda.current_stream(dev).wait_stream(comm_stream)
    ev_end.record()
    sync_all()
    clocks = None
    if rank == 0:
        try:
            clocks = sampler.stop()
        except Exception as exc:
            clocks = {"sm_mhz": None, "sm_max_mhz": None, "reasons": [f"sampler failed: {type(exc).__name__}"], "samples": 0}
    total_ms = ev[0].elapsed_time(ev_end)
    step_ms = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(args.steps))
    t = torch.tensor([total_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    total_ms = float(t.item())
    ms_per_step = total_ms / args.steps
    value = world * n_local * args.steps / (total_ms / 1e3)
    boxes, scores, labels, counts, status = out
    if args.dump_outputs and rank == 0:
        import numpy as np

        os.makedirs(args.dump_outputs, exist_ok=True)
        # slots past an image's count are never written by the NMS kernel: zero them so that the files depend only on
        # the detections
        valid = torch.arange(boxes.shape[1], device=boxes.device)[None, :] < counts.view(-1, 1)
        for name, t in (("boxes", boxes), ("scores", scores), ("labels", labels)):
            t = t.detach().float()
            t = torch.where(valid.view(*valid.shape, *([1] * (t.dim() - 2))), t, torch.zeros((), device=t.device))
            np.save(os.path.join(args.dump_outputs, f"{name}.npy"), t.cpu().numpy())
        np.save(os.path.join(args.dump_outputs, "counts.npy"), counts.detach().float().cpu().numpy())
    st = status.cpu().tolist()
    cand_per_img = st[0] / n_local
    det_per_img = float(counts.float().mean().item())

    # ---- per-stage leg (rank 0's own GPU; separate from the headline loop so that the event records do not perturb
    # it): CUDA events around letterbox | plan | counter init | decode | NMS of every step ---------------------------
    from yolort_b200 import _C

    stage_names = ("letterbox", "plan", "begin", "decode", "nms")
    stage_t = {k: [] for k in stage_names}
    marks = []

    def mark(_name=None):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        marks.append(e)

    pc = model.model.post_config()
    for i in range(min(args.steps, 20) + 2):
        marks.clear()
        ims_i = dev_lists[i % NBUF]
        # keep the GPU busy (~2 ms spin) while the host enqueues the stages, so that the events bracket GPU execution
        # only -- with an idle queue the first interval would include the host's own launch latency
        torch.cuda._sleep(4_000_000)
        mark()
        plan_i, rescale = model._prepare(ims_i)
        mark()
        plan_i.run()
        mark()
        _C.decode_nms_padded(plan_i.heads, "nhwc", pc["strides"], pc["anchors_px"], pc["num_classes"], pc["score_thresh"],
                             pc["nms_thresh"], pc["detections_per_img"], pc["semantics"], rescale, stage_hook=mark)
        torch.cuda.synchronize(dev)
        if i >= 2:
            for k, name in enumerate(stage_names):
                stage_t[name].append(marks[k].elapsed_time(marks[k + 1]) * 1e3)
    plan_us = median(stage_t["plan"])
    plan_ms = plan_us / 1e3
    src_bytes = h2d_bytes                                   # 3*h*w uint8 per image
    hb_wb = [(p.H, p.W) for p in engine._plans.values()]
    canvas_px = sum(h * w for h, w in hb_wb) / len(hb_wb)
    lb_bytes = src_bytes + n_local * 3 * canvas_px * 2      # SURVEY.md 8d: 3*Hs*Ws read + 3*Hb*Wb*2 written
    anchors = sum(int(hd.shape[1]) * int(hd.shape[2]) for hd in plan_i.heads) * pc["n_anchors"]
    dec_bytes = n_local * anchors * (pc["num_classes"] + 5) * 2    # SURVEY.md 8d: the head logits, read once

    # ---- heavier post-processing load: one short loop at a lower score threshold (~10x the candidates) ----------------
    heavy = None
    if args.config == "c2" and args.score_thresh is None and world == 1:
        HEAVY_THR = 0.12
        model.model.post_process.score_thresh = HEAVY_THR
        model(dev_lists[0])              # the list API grows the candidate arena when an image overflows its share
        for i in range(3):
            out_h = step_device(i)
        sync_all()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(10):
            out_h = step_device(i)
        e1.record()
        sync_all()
        st_h = out_h[4].cpu().tolist()
        heavy = {"score_thresh": HEAVY_THR, "candidates_per_image": st_h[0] / n_local, "ms_per_step": e0.elapsed_time(e1) / 10,
                 "images_per_s": n_local * 10 / (e0.elapsed_time(e1) / 1e3), "arena_overflow": int(st_h[1])}
        model.model.post_process.score_thresh = thr

    # ---- end-to-end leg through the public API, host tensors -----------------------------------------------
    e2e = None
    if not args.no_e2e:
        for i in range(3):
            model.predict(host_lists[i % NBUF])
        sync_all()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        d2h = 0
        t0 = time.perf_counter()
        e0.record()
        for i in range(args.steps):
            dets = model.predict(host_lists[i % NBUF])          # H2D of the uint8 images inside
            # D2H of the results: one copy per field (scores / labels / boxes of the whole batch)
            host_out = {k: torch.cat([d[k] for d in dets]).cpu() for k in ("scores", "labels", "boxes")}
            if i == 0:
                d2h = sum(v.numel() * v.element_size() for v in host_out.values()) + 4 * n_local + 32
        e1.record()
        sync_all()
        e2e_ms = max(e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3)
        t = torch.tensor([e2e_ms], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        e2e_sync_value = world * n_local * args.steps / (float(t.item()) / 1e3)
        d2h_sync = int(d2h)

        # throughput API: YOLOv5.predict_stream over the same host batches.  Every step's H2D (pinned host memory) and
        # D2H (padded detections) is inside the timed region; the API overlaps the copy of batch i+1 with the compute
        # of batch i (two batches in flight).
        e2e_value, e2e_api, d2h, stream_err = e2e_sync_value, "YOLOv5.predict(list of host tensors)", d2h_sync, None
        sync_all()
        try:   # no collective inside the try: a rank that fails must not leave the others waiting in a barrier
            for _ in model.predict_stream(host_lists[i % NBUF] for i in range(3)):
                pass
            torch.cuda.synchronize(dev)
            n_out = 0
            t0 = time.perf_counter()
            e0.record()
            for dets in model.predict_stream(host_lists[i % NBUF] for i in range(args.steps)):
                n_out += len(dets)
            e1.record()
            torch.cuda.synchronize(dev)
            assert n_out == n_local * args.steps
            stream_ms = max(e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3)
        except Exception as exc:   # keep the line: fall back to the synchronous call's number
            stream_err = f"{type(exc).__name__}: {exc}"[:200]
            stream_ms = -1.0
        t = torch.tensor([stream_ms, -stream_ms], dtype=torch.float64, device=dev)   # max over ranks, and "any rank failed"
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if float(t[1].item()) < 0:      # every rank measured it
            e2e_value = world * n_local * args.steps / (float(t[0].item()) / 1e3)
            e2e_api = "YOLOv5.predict_stream(iterable of host batches), 2 batches in flight"
            d2h = n_local * D * 6 * 4 + (n_local + 4) * 8
        elif stream_err is None:
            stream_err = "another rank failed"
        e2e = {"value": e2e_value, "unit": "images/s", "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": int(d2h),
               "api": e2e_api,
               "sync_call": {"value": e2e_sync_value, "api": "YOLOv5.predict(list of host tensors)", "d2h_bytes_per_step": d2h_sync},
               **({"stream_error": stream_err} if stream_err else {})}

    if rank == 0:
        sm = (clocks or {}).get("sm_mhz")
        peak, hbm, peak_src = measured_peaks(sm, (clocks or {}).get("sm_max_mhz"))
        flops = n_local * GFLOP_PER_IMAGE[cfg["model"]] * 1e9 * (canvas_px / (640.0 * 640.0))
        achieved = flops / (plan_ms / 1e3) / 1e12
        n_ops = plan_i.plan.n_ops

        def stage(name, nbytes):
            us = median(stage_t[name])
            d = {"us": us}
            if nbytes:
                d.update({"algorithmic_bytes": int(nbytes), "achieved_gbs": nbytes / us / 1e3, "frac_of_hbm": nbytes / us / 1e3 / hbm})
            return d

        line = {
            "metric": "images/sec end-to-end (letterbox->NMS)", "value": value, "unit": "images/s", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "p50_ms": step_ms[len(step_ms) // 2],
            "higher_is_better": True, "scaling": scaling, "vs_baseline": None, "dtype": cfg["dtype"], "data": "synthetic",
            "config": {"workload": cfg["what"], "name": args.config, "images_per_gpu_per_step": n_local,
                       "score_thresh": thr, "nms_thresh": 0.45, "detections_per_img": D,
                       "candidates_per_image": cand_per_img, "detections_per_image": det_per_img,
                       "distinct_canvases": n_canvases,
                       "l2": f"{NBUF} rotating input batches of {h2d_bytes / 1e6:.1f} MB (> 50 MB L2 in total); the activations of a step evict everything",
                       "parallelism": f"dp{world}" + (" + one nccl all_gather of the packed detections per step (side stream)" if world > 1 else "")},
            "gpu_launches": (n_ops + 1 + 3) * args.steps,
            "roofline": {"bound": "tensor", "achieved": achieved, "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak,
                         "peak_source": peak_src,
                         "kernel": "conv_wgmma_kernel + conv3x3_patch_kernel (all conv launches of one step)",
                         "plan_ms": plan_ms, "launches_per_step": n_ops, "arena_bytes": plan_i.arena_bytes},
            "roofline_stages": {"hbm_peak_gbs": hbm, "timing": "CUDA events around each stage, median over steps (separate loop)",
                                "letterbox": stage("letterbox", lb_bytes), "plan": stage("plan", 0),
                                "nms_begin": stage("begin", 0), "decode": stage("decode", dec_bytes), "nms": stage("nms", 0)},
            "clocks": clocks,
        }
        if e2e is not None:
            line["e2e"] = e2e
        if heavy is not None:
            line["nms_heavy_load"] = heavy
        if not args.no_cpu_baseline and world == 1:
            n_cpu = CPU_SAMPLE_IMAGES if size <= 640 else 1
            cpu_ims = [im.cpu() for im in dev_lists[0][:n_cpu]]
            ips, times, ref_dets = cpu_port_images_per_s(sd, 2, 1, cpu_ims, size=(size, size), thr=thr)
            line["cpu_baseline"] = {"value": ips, "unit": "images/s", "cores": torch.get_num_threads(), "kind": "port",
                                    "sample": f"{n_cpu} of the {n_local} images x 2 steps after 1 warm-up, fp32 oracle port"}
            # parity of THIS run: the GPU detections of the same images against the oracle's (north_star tolerance)
            try:
                sys.path.insert(0, os.path.join(ROOT, "tests"))
                import parity_util as util

                got = model(dev_lists[0])[:n_cpu]
                side = float(size) if not mixed else float(max(max(im.shape[-2:]) for im in cpu_ims))
                agg = {"n_ref": 0, "pairs": 0.0, "within": 0.0, "max_box_rel": 0.0, "max_score_err": 0.0}
                for g_, r_ in zip(got, ref_dets):
                    ps = util.pair_stats(util.to_np(g_), r_, side)
                    agg["n_ref"] += ps["n_ref"]
                    agg["pairs"] += ps["matched"] * ps["n_ref"]
                    agg["within"] += ps["within"] * ps["matched"] * ps["n_ref"]
                    agg["max_box_rel"] = max(agg["max_box_rel"], ps["max_box_rel"])
                    agg["max_score_err"] = max(agg["max_score_err"], ps["max_score_err"])
                line["parity"] = {"images": n_cpu, "oracle_detections": agg["n_ref"],
                                  "matched_fraction": agg["pairs"] / max(agg["n_ref"], 1),
                                  "boxes_within_1e-3_of_side": agg["within"] / max(agg["pairs"], 1),
                                  "max_box_err_over_side": agg["max_box_rel"], "max_score_err": agg["max_score_err"],
                                  "labels": "exact on matched pairs (label equality is part of the match)"}
            except Exception as exc:
                line["parity"] = {"error": f"{type(exc).__name__}: {exc}"[:200]}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
