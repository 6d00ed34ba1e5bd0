"""The statistics of tests/sample_stats.py on the CPU: they accept torch.multinomial draws from the distribution they
are given, reject draws made at a temperature 3 % off, and reject draws whose rows alias (a row repeating the stream
of the row before it).  Every draw uses a fixed seed, so every verdict is deterministic."""
import torch

from sample_stats import (chi2_sf, chi2_test, equal_streams, independence_test, kolmogorov_sf, ks_uniform,
                          merge_bins, prob_order, randomized_pit)

P_ACCEPT = 1e-6  # the bar of tests/test_gpu_sampling_f64.py: p >= this accepts
V = 626


def _logits(seed, V=V, scale=1.5):
    return torch.randn(V, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale


def _draws(probs, n, seed):
    return torch.multinomial(probs.float(), n, replacement=True, generator=torch.Generator().manual_seed(seed))


def test_chi2_sf_and_kolmogorov_tail_known_values():
    assert abs(chi2_sf(3.841458820694124, 1) - 0.05) < 1e-9
    assert abs(chi2_sf(18.307038053275146, 10) - 0.05) < 1e-9
    assert abs(kolmogorov_sf(1.3580986393225505) - 0.05) < 1e-6
    assert kolmogorov_sf(0.0) == 1.0 and kolmogorov_sf(10.0) < 1e-80


def test_merge_bins_each_group_expects_at_least_the_minimum():
    e = torch.tensor([0.1, 9.0, 0.5, 3.0, 4.0, 100.0, 0.2, 2.0])
    lab = merge_bins(e, 5.0)
    per = torch.zeros(int(lab.max()) + 1).index_add_(0, lab, e)
    assert (per >= 5.0).all(), per
    assert int(lab.max()) + 1 >= 3


def test_chi2_accepts_multinomial_and_rejects_a_perturbed_temperature():
    x = _logits(1)
    p = torch.softmax(x, -1)
    ids = _draws(p, 1 << 18, 2)
    stat, df, pv, out = chi2_test(ids, p)
    assert out == 0 and pv >= P_ACCEPT, (stat, df, pv)
    _, _, pw, _ = chi2_test(ids, torch.softmax(x / 1.03, -1))
    assert pw < P_ACCEPT, pw
    # draws made at the perturbed temperature, tested against the right distribution
    _, _, pd, _ = chi2_test(_draws(torch.softmax(x / 1.03, -1), 1 << 18, 3), p)
    assert pd < P_ACCEPT, pd


def test_chi2_counts_draws_outside_the_support():
    p = torch.softmax(_logits(4), -1)
    p[:10] = 0
    ids = _draws(p / p.sum(), 10000, 5)
    ids[:3] = 0
    assert chi2_test(ids, p / p.sum())[3] == 3


def test_pit_ks_accepts_multinomial_and_rejects_a_perturbed_temperature():
    g = torch.Generator().manual_seed(6)
    n = 20000
    lg = torch.randn(n, V, generator=g, dtype=torch.float64) * 1.5
    probs = torch.softmax(lg, -1)
    ids = torch.multinomial(probs, 1, generator=g)[:, 0]
    for order in (None, prob_order(probs)):  # id order and descending probability: both U(0, 1) for correct draws
        d, pv = ks_uniform(randomized_pit(probs, ids, torch.Generator().manual_seed(7), order))
        assert pv >= P_ACCEPT, (d, pv)
    alt = torch.softmax(lg / 1.05, -1)
    d2, pw = ks_uniform(randomized_pit(alt, ids, torch.Generator().manual_seed(7), prob_order(alt)))
    assert pw < P_ACCEPT, (d2, pw)


def test_ks_uniform_values():
    u = torch.rand(100000, generator=torch.Generator().manual_seed(8), dtype=torch.float64)
    assert ks_uniform(u)[1] >= P_ACCEPT
    assert ks_uniform(u ** 1.02)[1] < P_ACCEPT


def test_aliased_rows_are_rejected():
    """Uniform draws, 512 rows x 64 steps: independent rows pass; rows 2i + 1 repeating row 2i (a counter that drops
    its lowest row bit) give equal streams and fail the row r / r + 1 independence test."""
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, V, (512, 64), generator=g)
    assert equal_streams(ids) == [] and equal_streams(ids.T) == []
    assert independence_test(ids[:-1], ids[1:], V)[2] >= P_ACCEPT
    assert independence_test(ids[:, :-1], ids[:, 1:], V)[2] >= P_ACCEPT
    alias = ids.clone()
    alias[1::2] = alias[0::2]
    assert len(equal_streams(alias)) == 10  # 256 equal pairs, the first 10 listed
    assert independence_test(alias[0::2], alias[1::2], V)[2] < P_ACCEPT
    # a step the noise ignores: every step of a row repeats step 0
    still = ids[:, :1].expand(-1, 64)
    assert equal_streams(still.T) != []
    assert independence_test(still[:, :-1], still[:, 1:], V)[2] < P_ACCEPT
