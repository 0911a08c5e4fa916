"""predict_sharded on real devices (NCCL, one process per GPU) == the single-GPU forward on the same mixed-size batch.
Needs two H100s: python -m pytest tests/test_gpu_sharded.py -m gpu; skipped on a single-GPU machine."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import parity_util as util

pytestmark = pytest.mark.gpu

SIZES = [(97, 128), (128, 64), (75, 75), (50, 117), (128, 128), (100, 90), (64, 128)]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _build(dev):
    from yolort_b200.models import yolov5n

    sd = util.synth_state_dict(util.layouts()["n"], knob_obj=7.0, knob_cls=4.5, seed=0)
    m = yolov5n(size=(128, 128), score_thresh=0.15).eval()
    m.load_state_dict(sd)
    return m.to(dev)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device(f"cuda:{rank}")
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from yolort_b200.parallel import predict_sharded

        m = _build(dev)
        ims = [util.synth_image_u8(h, w, 40 + i) for i, (h, w) in enumerate(SIZES)]
        out = predict_sharded(m, ims)
        if rank == 0:
            q.put([{k: v.cpu() for k, v in d.items()} for d in out])
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two devices")
def test_predict_sharded_equals_single_gpu_forward():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    m = _build(torch.device("cuda:0"))
    ims = [util.synth_image_u8(h, w, 40 + i) for i, (h, w) in enumerate(SIZES)]
    want = m([im.to("cuda:0") for im in ims])
    assert len(got) == len(want) == len(SIZES)
    for g, w in zip(got, want):
        assert torch.equal(g["labels"], w["labels"].cpu())
        assert torch.equal(g["scores"], w["scores"].cpu()) and torch.equal(g["boxes"], w["boxes"].cpu())
