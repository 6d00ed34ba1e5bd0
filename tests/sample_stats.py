"""Goodness-of-fit statistics for sampled token ids, in float64 torch (no scipy).

* ``chi2_test``: Pearson chi-square of id counts against expected probabilities, the least likely bins merged until
  each merged bin expects at least ``min_expected`` draws; p from the regularized upper incomplete gamma function
  (``torch.special.gammaincc``).  Draws outside the expected support are counted apart (``outside``): the test makes
  no verdict on them, the caller asserts there are none.
* ``ks_uniform``: one-sample Kolmogorov-Smirnov test of values in [0, 1] against U(0, 1), with Stephens' small-sample
  correction of the statistic and the closed-form Kolmogorov tail ``2 sum_k (-1)^(k-1) exp(-2 k^2 x^2)``.
* ``randomized_pit``: the randomized probability integral transform of discrete draws, ``u = F(id - 1) + U p(id)``
  with F the cumulative distribution in id order.  If every id is drawn from its row's p, the u are i.i.d. U(0, 1).
* ``independence_test``: chi-square test of independence of two id sequences, each binned into ``bins`` classes.
* ``equal_streams``: pairs of identical rows of a [streams, draws] id table.

Every input is a tensor; every verdict is a number that a fixed seed makes deterministic.
"""
from __future__ import annotations

import math
from typing import List, Tuple

import torch


def chi2_sf(stat: float, df: int) -> float:
    """P(X >= stat) for X ~ chi-square with ``df`` degrees of freedom."""
    if df <= 0:
        return 1.0
    return float(torch.special.gammaincc(torch.tensor(df / 2.0, dtype=torch.float64),
                                         torch.tensor(stat / 2.0, dtype=torch.float64)))


def merge_bins(expected: torch.Tensor, min_expected: float = 5.0) -> torch.Tensor:
    """Group labels [n] for the bins of ``expected`` [n] (counts, > 0): bins in ascending order of expectation are
    merged into one group until the group expects at least ``min_expected``; a short last group joins the one before."""
    order = torch.argsort(expected, stable=True)
    label = torch.empty(expected.numel(), dtype=torch.long)
    g, acc = 0, 0.0
    e = expected[order].tolist()
    for j, i in enumerate(order.tolist()):
        label[i] = g
        acc += e[j]
        if acc >= min_expected and j < len(e) - 1:
            g, acc = g + 1, 0.0
    if acc < min_expected and g > 0:  # the largest bins end the order; a short tail group is merged back
        label[label == g] = g - 1
    return label


def chi2_test(ids: torch.Tensor, probs: torch.Tensor, min_expected: float = 5.0):
    """Pearson chi-square of ``ids`` (any shape, values in [0, V)) against ``probs`` [V] (sums to 1).
    Returns (stat, df, p, outside): ``outside`` counts draws where probs is 0; they are left out of the statistic."""
    probs = probs.to(torch.float64).cpu()
    V = probs.numel()
    counts = torch.bincount(ids.reshape(-1).long().cpu(), minlength=V).to(torch.float64)
    assert counts.numel() == V, "id out of range"
    sup = probs > 0
    outside = int(counts[~sup].sum())
    n = float(counts[sup].sum())
    exp = probs[sup] / probs[sup].sum() * n
    label = merge_bins(exp, min_expected)
    G = int(label.max()) + 1
    o = torch.zeros(G, dtype=torch.float64).index_add_(0, label, counts[sup])
    e = torch.zeros(G, dtype=torch.float64).index_add_(0, label, exp)
    stat = float(((o - e) ** 2 / e).sum())
    return stat, G - 1, chi2_sf(stat, G - 1), outside


def kolmogorov_sf(x: float) -> float:
    """P(K > x) for the Kolmogorov distribution: 2 sum_{k>=1} (-1)^(k-1) exp(-2 k^2 x^2)."""
    if x <= 0.0:
        return 1.0
    if x < 0.2:  # the alternating series converges slowly here, and the tail is 1 to double precision
        return 1.0
    s = 0.0
    for k in range(1, 101):
        t = math.exp(-2.0 * k * k * x * x)
        s += t if k % 2 else -t
        if t < 1e-300:
            break
    return min(1.0, max(0.0, 2.0 * s))


def ks_uniform(u: torch.Tensor) -> Tuple[float, float]:
    """Kolmogorov-Smirnov test of ``u`` against U(0, 1) -> (D, p)."""
    u = torch.sort(u.reshape(-1).to(torch.float64).cpu())[0]
    n = u.numel()
    i = torch.arange(1, n + 1, dtype=torch.float64)
    d = max(float((i / n - u).max()), float((u - (i - 1) / n).max()))
    sn = math.sqrt(n)
    return d, kolmogorov_sf(d * (sn + 0.12 + 0.11 / sn))


def randomized_pit(probs: torch.Tensor, ids: torch.Tensor, gen: torch.Generator, order: torch.Tensor = None
                   ) -> torch.Tensor:
    """``probs`` [n, V] (each row a distribution), ``ids`` [n] one draw per row -> u [n] float64:
    F(id - 1) + U p(id), U ~ U(0, 1) from ``gen``.  F is cumulative in id order, or in the token order ``order`` [n, V]
    (a permutation of 0 .. V - 1 per row) when given.  Any fixed order gives U(0, 1) for correct draws; ordering by
    descending probability (``prob_order``) turns a temperature error, which moves mass between likely and unlikely
    tokens, into one monotone deviation of the u, where id order scatters it across [0, 1] and it largely cancels."""
    probs = probs.to(torch.float64).cpu()
    ids = ids.reshape(-1, 1).long().cpu()
    if order is not None:
        order = order.cpu()
        probs = probs.gather(1, order)
        ids = torch.argsort(order, dim=-1).gather(1, ids)  # each id's position in its row's order
    cdf = probs.cumsum(-1)
    p = probs.gather(1, ids)[:, 0]
    below = cdf.gather(1, ids)[:, 0] - p
    U = torch.rand(ids.shape[0], generator=gen, dtype=torch.float64)
    return (below + U * p).clamp_(0.0, 1.0)


def prob_order(probs: torch.Tensor) -> torch.Tensor:
    """[n, V] -> each row's token ids by descending probability, ties by ascending id (an order for randomized_pit)."""
    return torch.argsort(-probs.to(torch.float64).cpu(), dim=-1, stable=True)


def independence_test(a: torch.Tensor, b: torch.Tensor, V: int, bins: int = 8):
    """Chi-square test of independence of paired ids ``a``, ``b`` (same shape, values in [0, V)), each binned into
    ``bins`` classes of consecutive ids -> (stat, df, p)."""
    x = (a.reshape(-1).long().cpu() * bins) // V
    y = (b.reshape(-1).long().cpu() * bins) // V
    t = torch.bincount(x * bins + y, minlength=bins * bins).to(torch.float64).view(bins, bins)
    r, c = t.sum(1, keepdim=True), t.sum(0, keepdim=True)
    keep_r, keep_c = r[:, 0] > 0, c[0] > 0
    t, r, c = t[keep_r][:, keep_c], r[keep_r], c[:, keep_c]
    e = r * c / t.sum()
    stat = float(((t - e) ** 2 / e).sum())
    df = (t.shape[0] - 1) * (t.shape[1] - 1)
    return stat, df, chi2_sf(stat, df)


def equal_streams(table: torch.Tensor) -> List[Tuple[int, int]]:
    """Pairs (i, j), i < j, of identical rows of the id table [streams, draws] (at most 10 listed)."""
    t = table.long().cpu()
    _, inv, cnt = torch.unique(t, dim=0, return_inverse=True, return_counts=True)
    pairs = []
    for g in torch.nonzero(cnt > 1)[:, 0].tolist():
        rows = torch.nonzero(inv == g)[:, 0].tolist()
        pairs += [(rows[0], r) for r in rows[1:]]
        if len(pairs) >= 10:
            break
    return pairs[:10]
