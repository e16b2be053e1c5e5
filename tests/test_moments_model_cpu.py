"""CPU model of the forward statistics scheme of csrc/syncbn.cu (`exchange_moments`): per strip Σ(r−s), Σ(r−s)² in fp32 with
s = the strip's first row → (mean, M2) per strip → fixed-order parallel-variance merge over strips, then over ranks.
Shows in fp32 arithmetic (numpy float32, the kernel's accumulation type) that the scheme keeps the variance where
E[x²] − E[x]² loses it, and that the merge is exact algebra (checked against float64 on the same data)."""
import numpy as np
import pytest

F = np.float32


def strip_moments(r: np.ndarray):
    """r: [rows, C] float32 rows of one strip → (n, mean[C], M2[C]) as the kernel forms them"""
    s = r[0].astype(F)
    d = (r - s).astype(F)
    s1 = d.sum(axis=0, dtype=F)
    s2 = (d * d).sum(axis=0, dtype=F)
    n = F(r.shape[0])
    mean = s + s1 / n
    m2 = np.maximum(s2 - s1 * (s1 / n), F(0))
    return n, mean.astype(F), m2.astype(F)


def merge(parts):
    """[(n, mean, M2)] → (N, mean, M2) in list order (hop 1b over strips, hop 2 over ranks)"""
    n_tot = F(sum(float(p[0]) for p in parts))
    mean = sum((p[0] * p[1] for p in parts), start=np.zeros_like(parts[0][1])) / n_tot
    m2 = sum((p[2] + p[0] * (p[1] - mean) ** 2 for p in parts), start=np.zeros_like(parts[0][2]))
    return n_tot, mean.astype(F), m2.astype(F)


@pytest.mark.parametrize("mean,std", [(100.0, 0.1), (-50.0, 1e-2), (1000.0, 1.0), (0.3, 1.5)])
@pytest.mark.parametrize("world", [1, 2, 8])
def test_strip_and_rank_merge_keeps_the_variance(mean, std, world):
    rng = np.random.default_rng(int(abs(mean) * 10) + world)
    C, rows, strips = 16, 6400, 37
    per_rank = []
    everything = []
    for _ in range(world):
        x = (rng.standard_normal((rows, C)) * std + mean).astype(F)
        everything.append(x)
        cuts = np.linspace(0, rows, strips + 1).astype(int)
        per_rank.append(merge([strip_moments(x[a:b]) for a, b in zip(cuts, cuts[1:])]))
    n, m, m2 = merge(per_rank)
    var = m2 / n
    x64 = np.concatenate(everything).astype(np.float64)
    np.testing.assert_allclose(m, x64.mean(axis=0), rtol=1e-6, atol=0)      # a few fp32 ulps of |mean|
    np.testing.assert_allclose(var, x64.var(axis=0), rtol=2e-4)
    # what the first-round kernel computed: E[x²] − E[x]² in fp32 — fine for mean ≈ std, useless for |mean| ≫ std
    x32 = np.concatenate(everything)
    naive = (x32 * x32).sum(axis=0, dtype=F) / F(x32.shape[0]) - (x32.sum(axis=0, dtype=F) / F(x32.shape[0])) ** 2
    err_naive = np.abs(naive - x64.var(axis=0)).max() / x64.var(axis=0).max()
    if abs(mean) / std >= 1000:
        assert err_naive > 1e-2
    if abs(mean) / std < 10:
        assert err_naive < 1e-4


def test_merge_is_independent_of_the_partition_up_to_rounding():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((5000, 8)) * 0.05 + 7.0).astype(F)
    ref = x.astype(np.float64).var(axis=0)
    for strips in (1, 2, 13, 132, 148):
        cuts = np.linspace(0, x.shape[0], strips + 1).astype(int)
        n, m, m2 = merge([strip_moments(x[a:b]) for a, b in zip(cuts, cuts[1:])])
        np.testing.assert_allclose(m2 / n, ref, rtol=3e-4)
