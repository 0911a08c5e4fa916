"""Device JPEG decode against torchvision's CPU decoder on one H100, in one process.

  * device decode of batches of 32 and 256 JPEGs at 640x480 (4:2:0, q75 and q95): the whole call (staging, one
    host-to-device copy, kernels; host clock ending in a synchronise, median over repeats), the same as compressed
    MB/s, and per kernel from a torch.profiler run of its own;
  * torchvision.io.decode_jpeg on the CPU over the same files, on 1, 8 and all host threads (host clock);
  * torchvision's nvJPEG decode_jpeg(device="cuda") as an outside reference point only;
  * predict(paths) img/s for bench.py's yolov5s workload at batch 32, device decode against YB_JPEG_DECODE=cpu,
    alternated, and whether the two give the same detections.
Prints the card name and power limit with the numbers and writes everything as JSON to --out.

    python scripts/jpeg_times.py --out jpeg_times.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import jpeg_corpus as J  # noqa: E402
from yolort_b200 import _C  # noqa: E402

DEV = torch.device("cuda:0")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def files(n, q):
    return [J.pil_jpeg(J.photo(480, 640, 10_000 * q + i), quality=q, subsampling=2) for i in range(n)]


def device_ms(datas, reps):
    """Host clock around one whole call (parse excluded: predict(paths) parses on its reader threads), staging, copy
    and kernels, ending in a synchronise."""
    infos = [_C.jpeg_parse(d) for d in datas]
    for _ in range(3):
        _C.jpeg_decode(datas, infos, DEV)
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t = time.perf_counter()
        _, status = _C.jpeg_decode(datas, infos, DEV)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1e3)
        assert not status.any()
    return statistics.median(times)


def kernel_us(datas, reps):
    """Device time per kernel, copy and memset of one call (torch.profiler, a run of its own)."""
    import re

    infos = [_C.jpeg_parse(d) for d in datas]
    _C.jpeg_decode(datas, infos, DEV)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            _C.jpeg_decode(datas, infos, DEV)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"jpeg_\w+_kernel|Memset|Memcpy \w+", e.key)
        t = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
        if m and t:
            out[m.group(0)] = out.get(m.group(0), 0) + round(t / reps, 1)
    out["total"] = round(sum(out.values()), 1)
    return out


def cpu_ms(datas, threads, reps):
    from torchvision.io import ImageReadMode, decode_jpeg

    blobs = [torch.frombuffer(bytearray(d), dtype=torch.uint8) for d in datas]

    def one(b):
        return decode_jpeg(b, mode=ImageReadMode.RGB)

    times = []
    with ThreadPoolExecutor(max_workers=threads) as pool:
        list(pool.map(one, blobs))
        for _ in range(reps):
            t = time.perf_counter()
            list(pool.map(one, blobs))
            times.append((time.perf_counter() - t) * 1e3)
    return statistics.median(times)


def nvjpeg_ms(datas, reps):
    from torchvision.io import ImageReadMode, decode_jpeg

    blobs = [torch.frombuffer(bytearray(d), dtype=torch.uint8) for d in datas]
    decode_jpeg(blobs, mode=ImageReadMode.RGB, device="cuda")
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t = time.perf_counter()
        decode_jpeg(blobs, mode=ImageReadMode.RGB, device="cuda")
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1e3)
    return statistics.median(times)


def predict_rates(paths, rounds, iters):
    model, _ = bench.build_model(bench.CONFIGS["c2"])       # bench.py's yolov5s workload: ~1000 candidates / image
    m = model.to(DEV)
    rates = {"gpu": [], "cpu": []}
    ingest = {"gpu": [], "cpu": []}
    for mode in ("gpu", "cpu"):                     # warm-up of both paths
        os.environ["YB_JPEG_DECODE"] = mode
        m.predict(paths)
    for _ in range(rounds):                         # the ingest alone: files -> device images, ending in a synchronise
        for mode in ("gpu", "cpu"):
            os.environ["YB_JPEG_DECODE"] = mode
            torch.cuda.synchronize()
            t = time.perf_counter()
            m._ingest_files(paths, DEV)
            torch.cuda.synchronize()
            ingest[mode].append(round((time.perf_counter() - t) * 1e3, 2))
    same = None
    for _ in range(rounds):
        for mode in ("gpu", "cpu"):
            os.environ["YB_JPEG_DECODE"] = mode
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(iters):
                out = m.predict(paths)
            torch.cuda.synchronize()
            rates[mode].append(len(paths) * iters / (time.perf_counter() - t))
            if mode == "gpu":
                g = out
            else:
                same = all(torch.equal(a["boxes"], b["boxes"]) and torch.equal(a["labels"], b["labels"])
                           for a, b in zip(g, out))
    os.environ.pop("YB_JPEG_DECODE")
    return {k: [round(v, 1) for v in r] for k, r in rates.items()}, ingest, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="jpeg_times.json")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    res = {"card": card(), "cpu_threads": os.cpu_count(), "decode": []}
    print("card:", res["card"], "| host threads:", res["cpu_threads"])
    for q in (75, 95):
        all_files = files(256, q)
        for n in (32, 256):
            datas = all_files[:n]
            mb = sum(len(d) for d in datas) / 1e6
            row = {"batch": n, "quality": q, "compressed_MB": round(mb, 2),
                   "device_ms": round(device_ms(datas, args.reps), 3)}
            row["device_MB_per_s"] = round(mb / row["device_ms"] * 1e3, 1)
            row["device_kernels_us"] = kernel_us(datas, 5)
            for t in sorted({1, 8, os.cpu_count()}):
                row[f"cpu_{t}_threads_ms"] = round(cpu_ms(datas, t, max(3, args.reps // 4)), 3)
            row["nvjpeg_reference_ms"] = round(nvjpeg_ms(datas, args.reps), 3)
            res["decode"].append(row)
            print(json.dumps(row))
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for i, d in enumerate(files(32, 75)):
            paths.append(os.path.join(tmp, f"{i}.jpg"))
            with open(paths[-1], "wb") as f:
                f.write(d)
        rates, ingest, same = predict_rates(paths, rounds=5, iters=10)
    res["predict_paths_yolov5s_b32"] = {"img_per_s": rates, "gpu_median": statistics.median(rates["gpu"]),
                                        "cpu_median": statistics.median(rates["cpu"]), "ingest_ms": ingest,
                                        "identical_detections": same}
    print(json.dumps(res["predict_paths_yolov5s_b32"]))
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
