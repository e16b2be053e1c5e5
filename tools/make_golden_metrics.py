#!/usr/bin/env python
"""Golden vectors for the evaluation metrics, produced by the UNMODIFIED reference classes
(utils/saliency_metric.py of the reference: CalTotalMetric and its five Cal* members) on seeded synthetic
prediction / ground-truth pairs normalised exactly as the reference's test loop does (train.py:396-409).
Writes tests/golden/metrics_kat.npz (inputs as uint8, per-image terms and the dataset dict).  Needs a checkout of the
reference (SOD_REFERENCE=/path/to/Distributed-SOD-Project); the tests only read the committed .npz."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.environ["SOD_REFERENCE"])
from utils.saliency_metric import CalTotalMetric  # noqa: E402


def cases():
    rng = np.random.default_rng(7)
    out = []
    for (h, w) in ((64, 64), (48, 80), (97, 61), (32, 32), (40, 40), (24, 56)):
        yy, xx = np.mgrid[0:h, 0:w]
        cy, cx, r = rng.uniform(0.2, 0.8) * h, rng.uniform(0.2, 0.8) * w, rng.uniform(0.15, 0.4) * min(h, w)
        disk = ((yy - cy) ** 2 + (xx - cx) ** 2) < r * r
        gt = (disk * rng.integers(128, 256)).astype(np.uint8)
        soft = 1 / (1 + np.exp(-(r - np.sqrt((yy - cy - 2) ** 2 + (xx - cx + 3) ** 2)) / 3.0))
        pred = np.clip(soft + rng.normal(0, 0.15, (h, w)), 0, 1)
        out.append(((pred * 255).astype(np.uint8), gt))
    h = w = 32
    out.append((np.full((h, w), 77, np.uint8), out[3][1].copy()))                      # constant prediction (max == min)
    out.append((rng.integers(0, 256, (h, w), dtype=np.uint8), np.zeros((h, w), np.uint8)))   # empty ground truth
    out.append((rng.integers(0, 256, (h, w), dtype=np.uint8), np.full((h, w), 255, np.uint8)))   # full ground truth
    out.append((np.zeros((h, w), np.uint8), out[3][1].copy()))                         # all-zero prediction
    return out


def main():
    cs = cases()
    total = CalTotalMetric(num=len(cs), beta_for_wfm=1)
    rec = {}
    for i, (p8, g8) in enumerate(cs):
        gt = g8 / (g8.max() + 1e-8)
        gt = np.where(gt > 0.5, 1, 0)
        mx, mn = p8.max(), p8.min()
        pred = p8 / 255 if mx == mn else (p8 - mn) / (mx - mn)
        total.update(pred, gt)
        rec[f"pred{i}"], rec[f"gt{i}"] = p8, g8
    rec["mae"] = total.cal_mae.prediction
    rec["meanf"] = total.cal_fm.meanF
    rec["precision"] = total.cal_fm.precision
    rec["recall"] = total.cal_fm.recall
    rec["sm"] = total.cal_sm.prediction
    rec["em"] = total.cal_em.prediction
    rec["wfm"] = total.cal_wfm.scores_list
    res = total.show()
    rec["show_keys"] = np.array(list(res))
    rec["show_vals"] = np.array([res[k] for k in res], dtype=np.float64)
    rec["n"] = np.array(len(cs))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "metrics_kat.npz"), **rec)
    print(res)


if __name__ == "__main__":
    main()
