"""Evaluation metrics seam: `CalTotalMetric` of the reference (utils/saliency_metric.py:306-341) with the per-pixel work
on the GPU and the evaluation distributed over the ranks (SURVEY §8f.4; the reference evaluates on rank 0 only and its
author lists multi-GPU evaluation as an open issue, readme.md:67-69).

How: after the reference's own normalisation (train.py:396-409) a prediction is k/D with integer k, D ≤ 255, and the
ground truth is binary — MAE, F-measure (adaptive meanF and the 255-bin PR curves behind maxF), S-measure and E-measure
are then functions of the joint histogram of (k, gt) over the four quadrants around the ground truth's centre of mass.
`csrc/pipeline.cu` produces those histograms with integer atomics (exact, order independent); the formulas below are the
reference's, evaluated in float64 on 2048 counters per image.  `show()` sums over the ranks with one all-reduce.

The weighted F-measure (utils/saliency_metric.py:232-303) needs an exact Euclidean distance transform and is the one
metric that is NOT a histogram functional.  `wfm="gpu"` runs it as three more kernels per batch (`csrc/wfm.cu`: scipy's
feature transform with its tie rule, then the 7×7 stencil and the weighted sums, reduced in a fixed order) and forms Q
from three float64 sums per image on the host; it agrees with the host path to 1e-10 per image.  `wfm="host"`
evaluates it with scipy on the rank's own images (same code path as the reference), `wfm=None` (default) leaves it
out of the result.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib

WFM_MODES = (None, "host", "gpu")


# ---- formulas on histograms (host, float64) -------------------------------------------------------------------------
def metrics_from_hist(hist: np.ndarray, head: np.ndarray, h: int, w: int) -> dict:
    """hist: uint[4,2,256] joint histogram (quadrant, gt, k); head: int64[8] = (min_u, max_u, max_gt, _, n_fg, Σy, Σx, _).
    Returns the per-image terms the reference's Cal* classes store (utils/saliency_metric.py)."""
    hist = hist.astype(np.float64)
    mn, mx, n_fg = int(head[0]), int(head[1]), int(head[4])
    n = float(h * w)
    d = mx - mn
    k = np.arange(256, dtype=np.float64)
    val = k / d if d > 0 else np.full(256, mn / 255.0)            # train.py:404-409 (only k = 0 is populated when d == 0)
    tot = hist.sum(axis=0)                                         # [2, 256]
    t0, t1 = tot[0], tot[1]
    all_k = t0 + t1
    mean_p = float((all_k * val).sum() / n)
    out = {}
    # MAE (utils/saliency_metric.py:70-71): |p - 0| on background, |p - 1| on foreground
    out["mae"] = float(((t0 * val).sum() + (t1 * (1.0 - val)).sum()) / n)
    # F-measure (utils/saliency_metric.py:17-54)
    th = min(2 * mean_p, 1)
    sel = val >= th
    if n_fg > 0:
        tp = float(t1[sel].sum())
        if tp == 0:
            meanf = 0.0
        else:
            pre, rec = tp / float(all_k[sel].sum()), tp / float(n_fg)
            meanf = 1.3 * pre * rec / (0.3 * pre + rec)
        p8 = np.uint8(val * 255).astype(np.int64)                  # np.uint8(pred * 255): truncation
        p8 = np.minimum(p8, 254)                                   # np.histogram(bins=range(256)): 255 falls into the last bin
        populated = all_k > 0
        th_t = np.bincount(p8[populated], weights=t1[populated], minlength=255)[:255]
        th_n = np.bincount(p8[populated], weights=t0[populated], minlength=255)[:255]
        t_cum, n_cum = np.cumsum(th_t[::-1]), np.cumsum(th_n[::-1])
        out["precision"] = t_cum / (t_cum + n_cum + 1e-8)
        out["recall"] = t_cum / float(n_fg)
        out["meanf"] = float(meanf)
    else:
        out["precision"], out["recall"], out["meanf"] = np.zeros(255), np.zeros(255), 0.0
    # S-measure (utils/saliency_metric.py:94-177)
    y = n_fg / n
    if y == 0:
        out["sm"] = 1 - mean_p
    elif y == 1:
        out["sm"] = mean_p
    else:
        def s_object(cnt, v):
            m = cnt.sum()
            x = (cnt * v).sum() / m
            s = np.sqrt(max((cnt * (v - x) ** 2).sum() / m, 0.0))
            return 2 * x / (x * x + 1 + s + 1e-8)
        obj = y * s_object(t1, val) + (1 - y) * s_object(t0, 1.0 - val)
        cy = int(round(int(head[5]) / n_fg)) + 1
        cx = int(round(int(head[6]) / n_fg)) + 1
        sizes = (cy * cx, cy * (w - cx), (h - cy) * cx, (h - cy) * (w - cx))      # LT, RT, LB, RB
        reg = 0.0
        for q in range(4):
            nq = float(sizes[q])
            if nq <= 0:
                continue                                            # empty quadrant: weight 0 (the reference yields nan here)
            c0, c1 = hist[q, 0], hist[q, 1]
            cq = c0 + c1
            x = (cq * val).sum() / nq
            # the reference casts the ground-truth quadrant to float32 before its mean / variance
            # (utils/saliency_metric.py:159): the mean of a 0/1 map is then the float32 quotient of two exact integers
            yq = float(np.float32(c1.sum()) / np.float32(nq))
            sx = (cq * (val - x) ** 2).sum() / nq
            sy = yq * (1 - yq)
            sxy = ((c1 * (val - x)).sum() * (1 - yq) + (c0 * (val - x)).sum() * (0 - yq)) / (nq - 1) if nq > 1 else 0.0
            alpha, beta = 4 * x * yq * sxy, (x * x + yq * yq) * (sx + sy)
            score = alpha / (beta + 1e-8) if alpha != 0 else (1.0 if beta == 0 else 0.0)
            reg += nq / n * score
        out["sm"] = float(0.5 * obj + 0.5 * reg)
    # E-measure (utils/saliency_metric.py:192-229)
    fm1 = np.array([t0[sel].sum(), t1[sel].sum()])                  # FM == 1 pixels by gt
    fm0 = np.array([t0[~sel].sum(), t1[~sel].sum()])
    if n_fg == 0:
        enhanced_sum = fm0.sum()
    elif n_fg == n:
        enhanced_sum = fm1.sum()
    else:
        mu_f, mu_g = fm1.sum() / n, n_fg / n
        enhanced_sum = 0.0
        for f, cnts in ((1.0, fm1), (0.0, fm0)):
            for g in (0, 1):
                a_f, a_g = f - mu_f, g - mu_g
                align = 2.0 * (a_g * a_f) / (a_g * a_g + a_f * a_f + 1e-8)
                enhanced_sum += cnts[g] * (align + 1) ** 2 / 4
    out["em"] = float(enhanced_sum / (n - 1 + 1e-8))
    return out


class SaliencyMetrics:
    """`CalTotalMetric` surface (`update` / `show`), batched and on the GPU.  Every rank feeds its own images; `show()`
    reduces over the ranks.  `num` is optional (the reference pre-sizes arrays with it)."""

    def __init__(self, num: int | None = None, beta_for_wfm: int = 1, wfm: str | None = None, group=None):
        if wfm not in WFM_MODES:
            raise ValueError(f"wfm must be one of {WFM_MODES}, not {wfm!r}")
        self.num, self.beta, self.wfm_mode, self.group = num, beta_for_wfm, wfm, group
        # (head int64[N,8] device, hist uint32[N,4,2,256] device, h, w, raw maps (wfm="host") or WFM sums float64[N,4]
        # device (wfm="gpu") or None)
        self._pending: list = []
        self._sums = {k: 0.0 for k in ("mae", "meanf", "sm", "em", "wfm")}
        self._precision, self._recall = np.zeros(255), np.zeros(255)
        self._count = 0

    # -- GPU part ---------------------------------------------------------------------------------------------------
    @staticmethod
    def quantize(pred: torch.Tensor, apply_sigmoid: bool = False) -> torch.Tensor:
        """float map(s) in [0,1] (or logits with apply_sigmoid) → uint8 as `ToPILImage` does (train.py:392-394)"""
        if not pred.is_cuda:
            raise _lib.SodError("SaliencyMetrics works on CUDA tensors (no CPU fallback)")
        pred = pred.contiguous()
        out = torch.empty(pred.shape, dtype=torch.uint8, device=pred.device)
        rc = _lib.lib().sod_saliency_quantize(pred.data_ptr(), _lib.dtype_code(pred.dtype), out.data_ptr(), pred.numel(),
                                              int(apply_sigmoid), _lib.stream_ptr())
        _lib.check(rc, "sod_saliency_quantize")
        _lib.count_launch()
        return out

    def update_batch(self, pred_u8: torch.Tensor, gt_u8: torch.Tensor) -> None:
        """pred_u8, gt_u8: uint8 [N,H,W] (or [N,1,H,W]) on the GPU — the 8-bit prediction map and the 8-bit ground truth
        as read from disk (train.py:386-397); normalisation and binarisation happen in the kernels.  Asynchronous."""
        if not (pred_u8.is_cuda and gt_u8.is_cuda):
            raise _lib.SodError("SaliencyMetrics works on CUDA tensors (no CPU fallback)")
        if pred_u8.dtype != torch.uint8 or gt_u8.dtype != torch.uint8 or pred_u8.shape != gt_u8.shape:
            raise ValueError("update_batch expects two uint8 tensors of the same shape")
        h, w = pred_u8.shape[-2:]
        p = pred_u8.reshape(-1, h, w).contiguous()
        g = gt_u8.reshape(-1, h, w).contiguous()
        n = p.shape[0]
        head = torch.empty((n, 8), dtype=torch.int64, device=p.device)
        hist = torch.zeros((n, 4, 2, 256), dtype=torch.int32, device=p.device)
        lib, s = _lib.lib(), _lib.stream_ptr()
        _lib.check(lib.sod_saliency_head(p.data_ptr(), g.data_ptr(), n, h, w, head.data_ptr(), s), "sod_saliency_head")
        split = self._split(head)
        _lib.check(lib.sod_saliency_hist(p.data_ptr(), g.data_ptr(), n, h, w, head.data_ptr(), split.data_ptr(), hist.data_ptr(), s),
                   "sod_saliency_hist")
        _lib.count_launch(2)
        extra = (p, g) if self.wfm_mode == "host" else None
        if self.wfm_mode == "gpu":
            extra = wfm_sums(p, g, head)
        self._pending.append((head, hist, h, w, extra))

    def update_ragged(self, pred, gt) -> None:
        """pred, gt: `pipeline.Ragged` uint8 "L" batches with the same per-image sizes (the prediction already resized to
        its ground truth's size, `pipeline.resize_u8`).  Same statistics as `update_batch`, images of any sizes in one
        pair of launches.  Asynchronous."""
        if not (pred.data.is_cuda and gt.data.is_cuda):
            raise _lib.SodError("SaliencyMetrics works on CUDA tensors (no CPU fallback)")
        if pred.channels != 1 or gt.channels != 1 or not torch.equal(pred.hw, gt.hw):
            raise ValueError("update_ragged expects two single-channel ragged batches of the same sizes")
        if bool((pred.hw[:, 0].long() * pred.hw[:, 1].long() >= 2 ** 31).any()):
            raise _lib.SodError("update_ragged: images of 2^31 pixels or more are not supported")
        n = len(pred)
        head = torch.empty((n, 8), dtype=torch.int64, device=pred.data.device)
        hist = torch.zeros((n, 4, 2, 256), dtype=torch.int32, device=pred.data.device)
        lib, s = _lib.lib(), _lib.stream_ptr()
        p, g, off, hw = pred.data.data_ptr(), gt.data.data_ptr(), pred.off_d.data_ptr(), pred.hw_d.data_ptr()
        _lib.check(lib.sod_saliency_head_ragged(p, g, n, off, hw, head.data_ptr(), s), "sod_saliency_head_ragged")
        split = self._split(head)
        _lib.check(lib.sod_saliency_hist_ragged(p, g, n, off, hw, head.data_ptr(), split.data_ptr(), hist.data_ptr(), s),
                   "sod_saliency_hist_ragged")
        _lib.count_launch(2)
        extra = ([pred.image(i) for i in range(n)], [gt.image(i) for i in range(n)]) if self.wfm_mode == "host" else None
        if self.wfm_mode == "gpu":
            extra = wfm_sums_ragged(pred, gt, head)
        self._pending.append((head, hist, pred.hw[:, 0].tolist(), pred.hw[:, 1].tolist(), extra))

    @staticmethod
    def _split(head: torch.Tensor) -> torch.Tensor:
        # quadrant split = int(round(centre of mass)) + 1 (utils/saliency_metric.py:122-124); round-half-even like Python's
        nfg = head[:, 4].clamp_min(1).double()
        split = torch.stack([torch.round(head[:, 5].double() / nfg), torch.round(head[:, 6].double() / nfg)], dim=1).to(torch.int32) + 1
        return split.contiguous()

    def update(self, pred: torch.Tensor, gt: torch.Tensor) -> None:
        """single image, reference signature (utils/saliency_metric.py:314): uint8 maps as above"""
        self.update_batch(pred[None], gt[None])

    # -- host part --------------------------------------------------------------------------------------------------
    def _drain(self) -> None:
        for head, hist, h, w, extra in self._pending:
            head_h, hist_h = head.cpu().numpy(), hist.cpu().numpy().astype(np.int64)
            sums = extra.cpu().numpy() if isinstance(extra, torch.Tensor) else None
            for i in range(head_h.shape[0]):
                # h, w: one size for the whole batch, or one per image (ragged batches)
                m = metrics_from_hist(hist_h[i], head_h[i], h[i] if isinstance(h, list) else h, w[i] if isinstance(w, list) else w)
                for k in ("mae", "meanf", "sm", "em"):
                    self._sums[k] += m[k]
                self._precision += m["precision"]
                self._recall += m["recall"]
                if sums is not None:
                    self._sums["wfm"] += wfm_from_sums(*sums[i, :3], self.beta)
                elif extra is not None:
                    self._sums["wfm"] += _wfm_host(extra[0][i].cpu().numpy(), extra[1][i].cpu().numpy(), self.beta)
                self._count += 1
        self._pending.clear()

    def show(self) -> dict:
        """dataset means over ALL ranks' images — the dict of utils/saliency_metric.py:324-341"""
        self._drain()
        vec = np.concatenate([[self._count], [self._sums[k] for k in ("mae", "meanf", "sm", "em", "wfm")], self._precision, self._recall])
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(self.group) > 1:
            # NCCL reduces device tensors; a gloo group (CPU tests of this host logic) reduces host tensors
            dev = "cuda" if dist.get_backend(self.group) == "nccl" else "cpu"
            t = torch.tensor(vec, dtype=torch.float64, device=dev)
            dist.all_reduce(t, group=self.group)
            vec = t.cpu().numpy()
        num = vec[0]
        if self.num is not None and int(num) != self.num:
            raise AssertionError(f"{self.num}, {int(num)}")         # the reference asserts the same (e.g. :49)
        precision, recall = vec[6:261] / num, vec[261:516] / num
        f = 1.3 * precision * recall / (0.3 * precision + recall + 1e-8)
        return {"MaxF": float(f.max()), "MeanF": float(vec[2] / num), "WFM": float(vec[5] / num) if self.wfm_mode else None,
                "MAE": float(vec[1] / num), "SM": float(vec[3] / num), "EM": float(vec[4] / num)}


# ---- weighted F-measure ---------------------------------------------------------------------------------------------
def wfm_gaussian() -> np.ndarray:
    """the reference's 7×7 MATLAB-style Gaussian with σ = 5 (utils/saliency_metric.py:279-283), float64"""
    ax = np.arange(-3, 4, dtype=np.float64)
    k = np.exp(-(ax[None, :] ** 2 + ax[:, None] ** 2) / (2.0 * 5 * 5))
    k[k < np.finfo(k.dtype).eps * k.max()] = 0
    k /= k.sum()
    return k


_wfm_coef = None


def _wfm_coef_ptr() -> int:
    """host address of the 50 doubles the WFM kernels take: the Gaussian row-major, then log(0.5)/5"""
    global _wfm_coef
    if _wfm_coef is None:
        _wfm_coef = (ctypes.c_double * 50)(*np.concatenate([wfm_gaussian().reshape(-1), [np.log(0.5) / 5]]).tolist())
    return ctypes.addressof(_wfm_coef)


def _wfm_call(entry: str, n: int, hw_host: torch.Tensor, args_before: tuple, nearest: torch.Tensor | None, device):
    hw_host = hw_host.to(torch.int32).contiguous()
    lib = _lib.lib()
    hw_p = hw_host.data_ptr()
    ws_bytes = lib.sod_saliency_wfm_workspace_bytes(n, hw_p)
    if ws_bytes == 0:
        raise _lib.SodError("WFM: image sizes must be positive, below 2^31 pixels and at most 2^21 wide")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    sums = torch.empty((n, 4), dtype=torch.float64, device=device)
    near = 0 if nearest is None else nearest.data_ptr()
    rc = getattr(lib, entry)(*args_before, _wfm_coef_ptr(), ws.data_ptr(), ws_bytes, sums.data_ptr(), near, _lib.stream_ptr())
    _lib.check(rc, entry)
    _lib.count_launch()
    return sums


def _check_nearest(nearest, px: int, device):
    if nearest is not None and (nearest.dtype != torch.int32 or not nearest.is_contiguous() or nearest.numel() != 2 * px
                                or nearest.device != device):
        raise ValueError("nearest: a contiguous int32 tensor of 2 × (total pixels) on the images' device")


def wfm_sums(pred_u8: torch.Tensor, gt_u8: torch.Tensor, head: torch.Tensor, nearest: torch.Tensor | None = None) -> torch.Tensor:
    """the weighted F-measure's per-image sums {ΣEw[gt], ΣEw[~gt], n_fg, 0} (float64 [N, 4], on the device) of equal-size
    uint8 maps [N, H, W] with `head` from sod_saliency_head; `nearest` (int32 [N, H, W, 2], optional) receives scipy's
    nearest-foreground (y, x) of every pixel.  Asynchronous."""
    if not (pred_u8.is_cuda and gt_u8.is_cuda and head.is_cuda):
        raise _lib.SodError("wfm_sums works on CUDA tensors (no CPU fallback)")
    n, h, w = pred_u8.shape
    _check_nearest(nearest, n * h * w, pred_u8.device)
    hw = torch.tensor([[h, w]] * n, dtype=torch.int32)
    return _wfm_call("sod_saliency_wfm", n, hw, (pred_u8.data_ptr(), gt_u8.data_ptr(), n, h, w, head.data_ptr()), nearest,
                     pred_u8.device)


def wfm_sums_ragged(pred, gt, head: torch.Tensor, nearest: torch.Tensor | None = None) -> torch.Tensor:
    """`wfm_sums` of two `pipeline.Ragged` "L" batches of the same sizes; `nearest`: int32 [Σ h·w, 2], images back to
    back.  Asynchronous."""
    if not (pred.data.is_cuda and gt.data.is_cuda and head.is_cuda):
        raise _lib.SodError("wfm_sums_ragged works on CUDA tensors (no CPU fallback)")
    n = len(pred)
    _check_nearest(nearest, int((pred.hw[:, 0].long() * pred.hw[:, 1].long()).sum()), pred.data.device)
    args = (pred.data.data_ptr(), gt.data.data_ptr(), n, pred.off_d.data_ptr(), pred.hw_d.data_ptr(), pred.hw.data_ptr(),
            head.data_ptr())
    return _wfm_call("sod_saliency_wfm_ragged", n, pred.hw, args, nearest, pred.data.device)


def wfm_from_sums(s_fg: float, s_bg: float, n_fg: float, beta: int = 1, eps: float = 1e-6) -> float:
    """Q of utils/saliency_metric.py:292-301 from one image's sums, in float64 as `_wfm_host` forms it (0 without
    foreground)"""
    if n_fg == 0:
        return 0.0
    tpw = n_fg - s_fg
    r = 1 - s_fg / n_fg
    p = tpw / (eps + tpw + s_bg)
    return float((1 + beta) * r * p / (eps + r + beta * p))


def _wfm_host(pred_u8: np.ndarray, gt_u8: np.ndarray, beta: int = 1, eps: float = 1e-6) -> float:
    """weighted F-measure of one image on the host (utils/saliency_metric.py:255-299): the distance transform keeps it off
    the histogram path; same scipy routines as the reference."""
    from scipy.ndimage import convolve, distance_transform_edt
    gt = gt_u8 / (gt_u8.max() + 1e-8) > 0.5
    mx, mn = int(pred_u8.max()), int(pred_u8.min())
    pred = pred_u8 / 255 if mx == mn else (pred_u8.astype(np.float64) - mn) / (mx - mn)
    if not gt.any():
        return 0.0
    dst, idx = distance_transform_edt(~gt, return_indices=True)
    err = np.abs(pred - gt)
    et = err.copy()
    et[~gt] = err[idx[0][~gt], idx[1][~gt]]
    k = wfm_gaussian()
    ea = convolve(et, weights=k, mode="constant", cval=0)
    min_e = np.where(gt & (ea < err), ea, err)
    ew = min_e * np.where(gt, 1.0, 2 - np.exp(np.log(0.5) / 5 * dst))
    tpw = gt.sum() - ew[gt].sum()
    fpw = ew[~gt].sum()
    r = 1 - ew[gt].mean()
    p = tpw / (eps + tpw + fpw)
    return float((1 + beta) * r * p / (eps + r + beta * p))
