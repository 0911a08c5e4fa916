"""Reproducible synthetic upstream checkpoints (tests/golden/upstream_ckpt_*.npz, written by
oracle/make_golden_checkpoint.py).

A torch checkpoint is a zip archive: `data.pkl` (the pickled object graph, which names the upstream classes
`models.yolo.*` / `models.common.*` and refers to tensor storages by key) plus one `data/<key>` record per storage.
The fixture keeps the skeleton and the small records verbatim; the large fp16 records (the conv weights) are
regenerated from a seed, so a multi-MB checkpoint fits in a few hundred KB and needs nothing outside the repository."""
import hashlib
import json
import pickle
import zipfile

import numpy as np
import torch

_RAW_MAX = 1024   # records up to this many bytes are stored verbatim (BN vectors, anchors, strides)
_DTYPES = {"HalfStorage": torch.float16, "FloatStorage": torch.float32, "DoubleStorage": torch.float64,
           "LongStorage": torch.int64, "IntStorage": torch.int32, "BoolStorage": torch.bool, "ByteStorage": torch.uint8}


class _Any:
    """Stand-in for every class named by the skeleton (only the storage records are of interest here)."""

    def __init__(self, *a, **k):
        pass

    def __setstate__(self, state):
        pass

    def __setitem__(self, k, v):
        pass

    def append(self, v):
        pass

    def extend(self, v):
        pass


class _StorageScan(pickle.Unpickler):
    def __init__(self, f):
        super().__init__(f)
        self.records = {}

    def find_class(self, module, name):
        return type(name, (_Any,), {"_name": name})

    def persistent_load(self, pid):
        # ('storage', storage_type, key, location, numel)
        self.records[str(pid[2])] = getattr(pid[1], "_name", str(pid[1]))
        return None


def _regen(seed: int, key: str, numel: int) -> bytes:
    g = torch.Generator().manual_seed(seed * 1000003 + int(key))
    return (torch.randn(numel, generator=g) * 0.05).half().numpy().tobytes()


def make_fixture(raw_path: str, seed: int) -> dict:
    """Arrays for np.savez: the archive's non-storage entries verbatim, and its storage records verbatim or regenerated."""
    with zipfile.ZipFile(raw_path) as z:
        names = z.namelist()
        pkl = next(n for n in names if n.endswith("/data.pkl"))
        prefix = pkl[: -len("data.pkl")]
        import io

        scan = _StorageScan(io.BytesIO(z.read(pkl)))
        scan.load()
        entries, out = [], {}
        for i, n in enumerate(names):
            data = z.read(n)
            if n.startswith(prefix + "data/"):
                key = n[len(prefix + "data/"):]
                stype = scan.records[key]
                if len(data) > _RAW_MAX and _DTYPES[stype] == torch.float16:
                    entries.append([n, "seeded", len(data) // 2, key])
                    continue
            entries.append([n, "raw", len(data), f"e{i}"])
            out[f"e{i}"] = np.frombuffer(data, dtype=np.uint8)
    out["entries"] = np.frombuffer(json.dumps({"seed": seed, "entries": entries}).encode(), dtype=np.uint8)
    return out


def rebuild_checkpoint(fixture, path: str) -> str:
    meta = json.loads(bytes(np.asarray(fixture["entries"])).decode())
    with zipfile.ZipFile(path, "w", zipfile.ZIP_STORED) as z:
        for name, mode, n, ref in meta["entries"]:
            data = _regen(meta["seed"], ref, n) if mode == "seeded" else bytes(np.asarray(fixture[ref]))
            z.writestr(name, data)
    return path


def describe(conv: dict) -> dict:
    """What a converter returned, in a form that can be stored and compared exactly."""
    sd = conv["state_dict"]
    return {"num_classes": int(conv["num_classes"]), "strides": [int(s) for s in torch.as_tensor(conv["strides"]).tolist()],
            "anchor_grids": [[float(x) for x in row] for row in conv["anchor_grids"]],
            "keys": list(sd.keys()),
            "tensors": {k: [str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().cpu().numpy().tobytes()).hexdigest()]
                        for k, v in sd.items()}}
