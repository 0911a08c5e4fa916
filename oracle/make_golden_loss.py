"""Writes tests/golden/loss.npz and loss.json: the unmodified reference SetCriterion (yolort/models/box_head.py:85-325)
on the cases of tests/loss_cases.py.  The inputs are regenerated from their seeds; only outputs are stored:

    <case>/<call>/losses        fp32 [3]: cls_logits, bbox_regression, objectness
    <case>/<call>/balance       fp64 [L]: `balance` after the call
    <case>/<call>/<level>/idx   int64 [M, 5]: b, a, gj, gi, class of each match, in the reference's order
    <case>/<call>/<level>/tbox, anchor     fp32 [M, 4], [M, 2]
    <case>/<call>/<level>/grad  fp32 [M, K]: the gradient at the matched cells, channels 0-3 from bbox_regression
                                alone, 4 from objectness alone, 5.. from cls_logits alone
    <case>/<call>/<level>/dense fp32 [S]: the objectness gradient at tests/loss_cases.dense_sample's cells

    python oracle/make_golden_loss.py
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import loss_cases as LC  # noqa: E402
from oracle.ref_import import import_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def main():
    import_reference()
    from yolort.models.box_head import SetCriterion

    arrays, meta = {}, {}
    for name, case in LC.cases().items():
        crit = SetCriterion(**case["kw"])
        meta[name] = {"kw": case["kw"], "calls": []}
        for k, (targets, heads) in enumerate(case["calls"]):
            heads = [h.clone().requires_grad_(True) for h in heads]
            L = len(heads)
            anchors = torch.as_tensor(crit.anchor_grids, dtype=torch.float32).view(L, -1, 2)
            anchors = anchors / torch.as_tensor(crit.strides, dtype=torch.float32).view(-1, 1, 1)
            cls_t, box_t, indices, anch = crit.build_targets(targets, heads, anchors)
            losses = crit(targets, heads)
            keys = ("cls_logits", "bbox_regression", "objectness")
            assert list(losses) == list(keys)
            grads = {}
            for key in keys:
                if not losses[key].requires_grad:        # no match: the term is a constant zero
                    grads[key] = [torch.zeros_like(h) for h in heads]
                    continue
                g = torch.autograd.grad(losses[key], heads, retain_graph=True, allow_unused=True)
                grads[key] = [torch.zeros_like(h) if x is None else x for x, h in zip(g, heads)]
            p = f"{name}/{k}"
            arrays[p + "/losses"] = np.array([float(losses[key]) for key in keys], np.float32)
            arrays[p + "/balance"] = np.array(crit.balance, np.float64)
            for i, h in enumerate(heads):
                b, a, gj, gi = indices[i]
                q = f"{p}/{i}"
                arrays[q + "/idx"] = torch.stack([b, a, gj, gi, cls_t[i]], 1).numpy().astype(np.int64)
                arrays[q + "/tbox"] = box_t[i].detach().numpy().astype(np.float32)
                arrays[q + "/anchor"] = anch[i].numpy().astype(np.float32)
                g = torch.cat([grads["bbox_regression"][i][..., :4], grads["objectness"][i][..., 4:5],
                               grads["cls_logits"][i][..., 5:]], -1)
                for key, lo, hi in (("bbox_regression", 4, None), ("objectness", 0, 4), ("cls_logits", 0, 5)):
                    other = grads[key][i]        # each component reaches only its own channels
                    assert float(other[..., lo:hi].abs().max()) == 0.0 if other.numel() else True
                arrays[q + "/grad"] = g[b, a, gj, gi].detach().numpy().astype(np.float32)
                cells = LC.dense_sample(h.shape)
                arrays[q + "/dense"] = g[..., 4].reshape(-1)[cells].detach().numpy().astype(np.float32)
            meta[name]["calls"].append({"n_targets": int(targets.shape[0]),
                                        "matches": [int(ix[0].numel()) for ix in indices],
                                        "losses": [float(losses[key]) for key in keys],
                                        "balance": list(crit.balance)})
    np.savez_compressed(os.path.join(OUT, "loss.npz"), **arrays)
    with open(os.path.join(OUT, "loss.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", os.path.join(OUT, "loss.npz"), len(arrays), "arrays")


if __name__ == "__main__":
    main()
