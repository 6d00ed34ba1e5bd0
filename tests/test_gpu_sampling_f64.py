"""The sampling tail - k_sample<false|true> (csrc/sampler.cu) and k_flow's in-kernel fl_sample_row (csrc/flow.cuh) -
against the distribution it should draw from, in float64.

A. Stand-alone ctb_sample with device Philox noise (q_noise None, the default manual_seed=None path): one fixed logits
   row replicated over R rows (each row its own Philox counter) and drawn at 64 steps: 2^20 draws per codebook on the
   sort path (V = 626), 2^18 on the search path (V = 21,178).  Fewer leave some power checks near their bar.  The expected distribution is the oracle's filters applied to the
   fp32 logits, softmax in float64.  No draw may fall outside its support; a Pearson chi-square (tokens of like
   probability merged into about 64 bins, each expecting thousands of draws) must give p >= P_MIN; the same draws against the distribution at temperature x 1.03 must give
   p < P_MIN, which shows the sample is large enough to see an error of that size.  Uniform rows, no filters (the id is
   then the arg-min of the noise: Philox seen directly): ids uniform over 626 bins, no two rows' 64-step streams and no
   two steps' 64-row streams equal, seeds that differ in their high 32 bits give different streams, and contingency
   tables of step s / s + 1, row r / r + 1 and codebook q / q + 1 do not reject independence.
B. Unseeded ids on every decode path - k_flow with in-kernel sampling at B = 1, 2, k_flow with k_sample
   (CTB_FLOW_NO_INK), k_step at B = 3, 8, the FMA chain at B = 6, the wgmma step at B = 12, fp32 slot engines at S = 4
   and 24 and a half-precision engine at S = 24, each engine with an unseeded text request (the 21,178-wide search
   path) - against the float64 model teacher-forced along the GPU's ids.  Every step's filtered float64 distribution
   is built.  Every id must lie in its support, except at steps whose top-p or top-k cut is within MARGIN of flipping
   (counted and printed as margin exceptions: on the 21,178-wide head some cumulative sum is always that close to the
   cut, so such steps cannot be left out of the statistics), EOS never before min_new_token, and the randomized
   probability integral transform of the ids over all steps must be
   uniform (Kolmogorov-Smirnov p >= P_MIN) while the same transform at temperature x 1.05 is rejected.  The transform
   orders each step's tokens by descending float64 probability (sample_stats.randomized_pit).
C. Seeded ids at the edges, exactly: both paths of k_sample against oracle.gpt_oracle.sample_step (the engine's
   k_sample<true> against the float64 teacher-forced model, k_flow's in-kernel sampler against k_sample through the
   two-handle comparison of test_gpu_small_batch_decode.py), at temperatures 1e-3 and 100, logits of +-1e4 and rows
   that underflow, -inf logits, top_p 1 and 1e-6, top_k 1 (min_keep 3), V - 1 and >= V, ties at the top-k cut, a
   penalty window of one id 31 times, negative penalized logits, the rows >= penalty_max_ids quirk, greedy ties, greedy
   with EOS the maximum, and an EOS ban that empties the row (id 0, as ATen's argmax of a NaN row).  An id may differ
   only where decision_margins is below MARGIN; each such exception is printed.  Three rules are the kernels' own and
   are tested against this file's restatement (``rule_sample``) instead of the oracle:
   1. a tie group at the top-p cut is kept whole (HF removes tied tokens by their position in torch.sort's output,
      an order that is not defined); the kept set contains the oracle's and differs only in tokens equal to the cut;
   2. -0.0 and +0.0 are one value at the top-k cut and the greedy maximum;
   3. top_k is used as given (TopKLogitsWarper has folded its own min_tokens_to_keep in); top-p's min_tokens_to_keep
      does not widen it.

Runs in about a minute on one H100 80 GB HBM3 (700 W), the float64 references included.
"""
import math
import zlib

import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.engine import EngineDevice, Request, schedule
from chattts_b200.processors import (ArgmaxOnly, CustomRepetitionPenaltyLogitsProcessorRepeat, TopKLogitsWarper,
                                     TopPLogitsWarper, build_sampler_config, gen_logits)
from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.sampler import sample_rows
from f64_oracle import F64Oracle, sample_trace
from gpu_util import expect_step, release_on_teardown
from oracle.gpt_oracle import (SamplerParams, apply_temperature, decision_margins, exp_noise, repetition_penalty,
                               sample_from_scores, sample_step, top_k_filter, top_p_filter)
from sample_stats import (chi2_test, equal_streams, independence_test, ks_uniform, prob_order, randomized_pit)
import test_gpu_small_batch_decode as sbd

pytestmark = pytest.mark.gpu

P_MIN = 1e-6
MARGIN = 1e-3
EOS, TEXT_EOS, V_CODE, V_TEXT = 625, 21001, 626, 21178
W16, KV16 = _lib.ENGINE_FP16_WEIGHTS, _lib.ENGINE_FP16_KV
INF = float("inf")

_oracles = {}
_release = release_on_teardown(_oracles, sbd._handles, sbd._weights, sbd._oracles, sbd._refs)


def _cfg(procs, temps, eos, min_new=0, philox=0):
    return build_sampler_config(procs, temps, eos, min_new, philox)


# ---------------------------------------------------------------------------------------------------- A
def _expected(logits, temps, procs, gen_rows):
    """float64 distribution [rows, V] of one item's rows (``logits`` [rpi, V] fp32): the oracle's filters on the fp32
    logits, softmax in float64."""
    x = apply_temperature(logits, torch.tensor(temps, dtype=torch.float32))
    for p in procs:
        if isinstance(p, CustomRepetitionPenaltyLogitsProcessorRepeat):
            x = repetition_penalty(gen_rows, x, p.penalty, p.max_input_ids, p.past_window)
        elif isinstance(p, TopPLogitsWarper):
            x = top_p_filter(x, p.top_p, p.min_tokens_to_keep)
        elif isinstance(p, TopKLogitsWarper):
            x = top_k_filter(x, p.top_k, 1)
    return torch.softmax(x.double(), -1)


def _draw(row, procs, temps, rpi, items, steps, philox, gen=None):
    """ids [steps, items, rpi] of ``row`` [V] replicated over items * rpi rows, device noise, steps 0 .. steps - 1."""
    V = row.numel()
    logits = row.float().reshape(1, V).expand(items * rpi, V).contiguous().cuda()
    cfg = _cfg(procs, temps, EOS if V == V_CODE else TEXT_EOS, 0, philox)
    g = None if gen is None else gen.expand(items, -1, -1).contiguous().cuda()
    out = torch.stack([sample_rows(logits, cfg, rpi, None, g, step=s) for s in range(steps)])
    return out.cpu().long().view(steps, items, rpi)


def _window(row, rpi, n_gen=20):
    """A repetition window [1, n_gen, rpi] of the row's 8 most likely ids, so that the penalty moves the distribution."""
    top = torch.topk(row, 8)[1]
    return top[torch.arange(n_gen) % 8].view(1, n_gen, 1).expand(1, n_gen, rpi).contiguous()


def _row(V, seed):
    """N(0, 1) logits with 64 tokens, at random positions, on a ramp from 8 down to -4.6: on the search path's 21,178
    tokens the top 20 of plain Gaussian logits are too alike for a 3 % temperature error to show in 2^16 draws."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(V, generator=g)
    x[torch.randperm(V, generator=g)[:64]] = 8.0 - 0.2 * torch.arange(64, dtype=torch.float32)
    return x


A_CASES = [  # (tag, processors, temperatures, rows per item, penalty window)
    ("none", (), [1.0], 1, False),
    ("p0.7_k20_rp1.05", (CustomRepetitionPenaltyLogitsProcessorRepeat(1.05, 10 ** 6, 16),
                         TopPLogitsWarper(0.7, 3), TopKLogitsWarper(20, 3)), [0.7], 1, True),
    ("p0.95", (TopPLogitsWarper(0.95, 3),), [1.0], 1, False),
    ("k20", (TopKLogitsWarper(20, 3),), [0.5], 1, False),
    ("rpi4_temps", (), [0.3, 0.7, 1.0, 1.5], 4, False),
]


# per-codebook rows are audio rows: the search path (text, one row per item) runs the others
A_PARAMS = [(c, V) for c in A_CASES for V in (V_CODE, V_TEXT) if c[3] == 1 or V == V_CODE]


@pytest.mark.parametrize("case,V", A_PARAMS, ids=[f"{c[0]}-{V}" for c, V in A_PARAMS])
def test_a_device_noise_draws_follow_the_distribution(case, V):
    tag, procs, temps, rpi, window = case
    draws = (1 << 20) if V == V_CODE else (1 << 18)  # per codebook: 2^18 / 2^16 leave the power check near its bar
    steps = 64
    items = draws // steps
    row = _row(V, 11 + V)
    gen = _window(row, rpi) if window else None
    ids = _draw(row, procs, temps, rpi, items, steps, philox=0x5EED0000 + V, gen=gen)
    one = row.reshape(1, V).expand(rpi, V).contiguous()
    gen_rows = gen[0].T if gen is not None else torch.zeros(rpi, 0, dtype=torch.long)
    want = _expected(one, temps, procs, gen_rows)
    alt = _expected(one, [t * 1.03 for t in temps], procs, gen_rows)
    for q in range(rpi):
        m = ids[:, :, q].numel() / 64  # about 64 bins of like probability: power against a smooth error
        stat, df, p, outside = chi2_test(ids[:, :, q], want[q], m)
        _, _, p_alt, out_alt = chi2_test(ids[:, :, q], alt[q], m)
        p_alt = 0.0 if out_alt else p_alt
        print(f"\nA {tag} V={V} q={q} T={temps[q]}: {ids[:, :, q].numel()} draws, support "
              f"{int((want[q] > 0).sum())}, chi2 {stat:.1f} df {df} p {p:.3g}; at T x 1.03 p {p_alt:.3g}")
        assert outside == 0, (tag, V, q, "draws outside the support", outside)
        assert p >= P_MIN, (tag, V, q, stat, df, p)
        assert p_alt < P_MIN, (tag, V, q, "not enough draws to see T x 1.03", p_alt)


def test_a_uniform_rows_show_philox_directly():
    """Zero logits, no filters: every id is the arg-min of its row's Exp(1) noise."""
    items, rpi, steps = 1024, 4, 64
    row = torch.zeros(V_CODE)
    ids = _draw(row, (), [1.0], rpi, items, steps, philox=0x1234_5678_9ABC)  # [steps, items, rpi]
    flat = ids.reshape(steps, items * rpi)  # [step, row]
    stat, df, p, outside = chi2_test(flat, torch.full((V_CODE,), 1.0 / V_CODE, dtype=torch.float64))
    print(f"\nA uniform: {flat.numel()} draws, chi2 {stat:.1f} df {df} p {p:.3g}")
    assert outside == 0 and p >= P_MIN, (stat, df, p)
    # a row's 64 steps, and a step's first 64 rows: no two streams equal (a step or row the counter ignores)
    assert equal_streams(flat.T) == [], equal_streams(flat.T)
    assert equal_streams(flat[:, :64]) == [], "two steps drew the same 64 rows"
    tests = {"step s / s+1": (flat[:-1], flat[1:]), "row r / r+1": (flat[:, :-1], flat[:, 1:]),
             "codebook q / q+1": (ids[:, :, :-1], ids[:, :, 1:])}
    for name, (a, b) in tests.items():
        st, d, pv = independence_test(a, b, V_CODE)
        print(f"A uniform {name}: chi2 {st:.1f} df {d} p {pv:.3g}")
        assert pv >= P_MIN, (name, st, d, pv)
    # seeds that differ only in their high 32 bits
    hi = _draw(row, (), [1.0], rpi, items, 1, philox=0x1234_5678_9ABC ^ (1 << 40))[0].reshape(-1)
    same = float((hi == flat[0]).double().mean())
    print(f"A uniform: seed ^ 2^40 repeats {same:.4f} of step 0's ids (1/626 = {1 / 626:.4f} expected)")
    assert same < 0.01, same


# ---------------------------------------------------------------------------------------------------- B
def _filtered(lg, ids, temps, top_p, top_k, rp, max_ids, eos, min_new, window=16):
    """float64 logits [n, rows, V] of a teacher-forced run and its ids [n, rows] -> (the filtered distribution each
    step's ids were drawn from [n, rows, V], float64; decision margin [n, rows] of the top-p and top-k cuts).  Step i's
    repetition window is ids[i - window : i]; steps before min_new ban EOS."""
    n, rows, V = lg.shape
    dev = lg.device
    x = lg / torch.tensor(temps, dtype=torch.float64, device=dev)[None, :, None]
    ids = ids.to(dev).long()
    if rp != 1.0:
        seen = torch.zeros(n + 1, rows, V, dtype=torch.int32, device=dev)
        seen[1:].scatter_(2, ids[:, :, None], 1)
        seen = seen.cumsum(0, dtype=torch.int32)  # seen[i]: counts over ids[:i]
        lo = (torch.arange(n, device=dev) - window).clamp(min=0)
        cnt = (seen[:n] - seen[lo]).double()
        cnt[:, max_ids:] = 0
        alpha = torch.pow(torch.tensor(rp, dtype=torch.float64, device=dev), cnt)
        del seen
        x = torch.where(x < 0, x * alpha, x / alpha)
    x = x.reshape(n * rows, V)
    margin = torch.full((n * rows,), INF, dtype=torch.float64, device=dev)
    if top_p is not None:
        cum = torch.sort(x, dim=-1)[0].softmax(-1).cumsum(-1)
        margin = torch.minimum(margin, (cum[:, :-3] - (1 - top_p)).abs().amin(-1))
        x = top_p_filter(x, top_p, 3)
    if top_k is not None:
        k = min(max(top_k, 3), V - 1)
        top = torch.topk(x, k + 1, dim=-1)[0]
        gap = (top[:, k - 1] - top[:, k]).nan_to_num(INF)
        margin = torch.minimum(margin, torch.where(torch.isfinite(top[:, k]), gap, INF))
        x = top_k_filter(x, top_k, 3)
    x = x.view(n, rows, V)
    x[: min(min_new, n), :, eos] = -INF
    return torch.softmax(x, -1), margin.view(n, rows)


def _pit_check(tag, runs, eos, min_new):
    """``runs``: list of (float64 logits [n, rows, V], ids [n, rows], temperatures, (top_p, top_k, rp, max_ids)).
    Support and EOS checks, then the PIT KS test and its power check over every run's kept steps together."""
    us, alts, exceptions, near, total = [], [], 0, 0, 0
    for lg, ids, temps, (tp, tk, rp, max_ids) in runs:
        ids = ids.long()
        n = ids.shape[0]
        assert not bool((ids[:min(min_new, n)] == eos).any()), (tag, "EOS before min_new_token")
        probs, margin = _filtered(lg, ids, temps, tp, tk, rp, max_ids, eos, min_new)
        alt, _ = _filtered(lg, ids, [t * 1.05 for t in temps], tp, tk, rp, max_ids, eos, min_new)
        tight = (margin < MARGIN).cpu()
        total += tight.numel()
        near += int(tight.sum())
        p_id = probs.gather(2, ids.to(probs.device)[:, :, None])[:, :, 0].cpu()
        bad = torch.nonzero(~tight & (p_id <= 0))
        assert bad.numel() == 0, (tag, "ids outside the support at (step, row)", bad[:8].tolist())
        exceptions += int((tight & (p_id <= 0)).sum())
        P, A, I = probs.cpu().flatten(0, 1), alt.cpu().flatten(0, 1), ids.flatten()
        seed = 1234 + len(us)
        us.append(randomized_pit(P, I, torch.Generator().manual_seed(seed), prob_order(P)))
        alts.append(randomized_pit(A, I, torch.Generator().manual_seed(seed), prob_order(A)))
    d, p = ks_uniform(torch.cat(us))
    d_alt, p_alt = ks_uniform(torch.cat(alts))
    print(f"\nB {tag}: {total} draws, {near} at steps within MARGIN of a cut, {exceptions} margin exceptions (id "
          f"outside the float64 support); KS D {d:.4f} p {p:.3g}; at T x 1.05 D {d_alt:.4f} p {p_alt:.3g}")
    assert exceptions <= total // 1000, (tag, exceptions, total)
    assert p >= P_MIN, (tag, d, p)
    assert p_alt < P_MIN, (tag, "not enough draws to see T x 1.05", d_alt, p_alt)


B_PARAMS = (0.5, None, 1.05)  # top-p 0.5 at low temperature: a 5 % temperature error is visible in ~10^4 draws
B_TEMPS = [0.3, 0.4, 0.4, 0.3]
B_DRAWS = 9000
# (tag, handle environment, max_batch, B, decode step)
STATIC = [("k_flow+ink B=1", sbd.INK_ENV, 2, 1, _lib.STEP_FLOW_INK),
          ("k_flow+ink B=2", sbd.INK_ENV, 2, 2, _lib.STEP_FLOW_INK),
          ("k_flow B=1 (CTB_FLOW_NO_INK)", sbd.EXT_ENV, 2, 1, _lib.STEP_FLOW),
          ("k_step B=3", sbd.STEP_ENV, 8, 3, _lib.STEP_MEGA),
          ("k_step B=8", sbd.STEP_ENV, 8, 8, _lib.STEP_MEGA),
          ("fma B=6", {"CTB_NO_FLOW": "1", "CTB_NO_MEGA": "1"}, 6, 6, _lib.STEP_FMA),
          ("wgmma B=12", {"CTB_GPT_TC": "1"}, 12, 12, _lib.STEP_WGMMA)]


def _f64(fp16=False):
    if fp16 not in _oracles:
        gs, es, _, _ = sbd._model("plain")
        _oracles[fp16] = F64Oracle(gs, es, fp16_layers=fp16, fp16_kv=fp16, device="cuda")
    return _oracles[fp16]


@pytest.mark.parametrize("case", STATIC, ids=[c[0] for c in STATIC])
def test_b_unseeded_static_batch_follows_float64(case):
    tag, env, max_batch, B, step = case
    max_new = math.ceil(B_DRAWS / (4 * B))
    lengths = [16 + 7 * b for b in range(B)]
    gpt, _ = sbd._gpt("plain", env, max_batch, 256 * math.ceil((max(lengths) + max_new + 1) / 256))
    expect_step(gpt, B, step)
    tp, tk, rp = B_PARAMS
    warp, proc = gen_logits(num_code=EOS, top_P=tp, top_K=tk, repetition_penalty=rp)
    outs, ids = sbd._generate(gpt, lengths, (*proc, *warp), B_TEMPS, max_new, max_new, None, pseed=70 + B,
                              philox=900 + B)
    got = outs[-1].ids
    orc = _f64()
    runs = []
    for b, L in enumerate(lengths):
        g = got[b].cpu()
        assert g.shape == (max_new, 4), (tag, b, g.shape)
        _, lg = orc.teacher_forced(orc.embed_prompt(ids[b, -L:]), g)
        runs.append((lg, g, B_TEMPS, (tp, tk, rp, EOS)))
    _pit_check(tag, runs, EOS, max_new)


ENGINES = [("fp32 S=4", 4, 0, 8), ("fp32 S=24", 24, 0, 24), ("fp16 S=24", 24, W16 | KV16, 24)]
TEXT_NEW = 1500


@pytest.mark.parametrize("case", ENGINES, ids=[c[0] for c in ENGINES])
def test_b_unseeded_engine_follows_float64(case):
    """Code requests and one text request (the search path), all unseeded, on one slot engine."""
    tag, slots, flags, n_code = case
    max_new = math.ceil(B_DRAWS / (4 * n_code))
    gpt, embed = sbd._gpt("plain", {}, 24, 2048)
    tp, tk, rp = B_PARAMS
    warp, proc = gen_logits(num_code=EOS, top_P=tp, top_K=tk, repetition_penalty=rp)
    twarp, tproc = gen_logits(num_code=V_TEXT, top_P=tp, top_K=tk, repetition_penalty=rp)
    prompts, reqs = [], []
    for i in range(n_code + 1):
        text = i == n_code
        L = 12 + 5 * i
        p = synth_prompt_batch([L], seed=300 + i)[0][0]
        prompts.append(p)
        emb = embed(p[None], torch.ones(1, L, dtype=torch.bool))[0]
        reqs.append(Request(emb=emb, temperature=[0.3] if text else B_TEMPS, eos_token=TEXT_EOS if text else EOS,
                            max_new_token=TEXT_NEW if text else max_new,
                            min_new_token=TEXT_NEW if text else max_new,
                            logits_processors=(*tproc, *twarp) if text else (*proc, *warp), infer_text=text))
    torch.manual_seed(4242 + slots + flags)  # the engine draws each request's Philox seed from torch's generator
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, TEXT_NEW, False, flags)
        for i, slot, n in schedule(reqs, dev, 64):
            got[i] = dev.harvest(slot, n).ids[0].cpu().clone()
    orc = _f64(bool(flags))
    runs = []
    for i in range(n_code):
        _, lg = orc.teacher_forced(orc.embed_prompt(prompts[i]), got[i])
        runs.append((lg, got[i], B_TEMPS, (tp, tk, rp, EOS)))
    _pit_check(f"engine {tag} codes", runs, EOS, max_new)
    t = got[n_code]
    assert t.shape == (TEXT_NEW,), t.shape
    _, lg = orc.teacher_forced_text(orc.embed_prompt(prompts[n_code]), t)
    _pit_check(f"engine {tag} text", [(lg, t[:, None], [0.3], (tp, tk, rp, V_TEXT))], TEXT_EOS, TEXT_NEW)


# ---------------------------------------------------------------------------------------------------- C
def rule_filter(x, top_p, p_min_keep, top_k):
    """The kernels' filters, restated: top-p keeps every token whose value is at least that of the smallest token HF
    keeps (ascending sort, ``cum <= 1 - top_p`` removed except the last ``p_min_keep``; the removed set is a prefix, so
    its length fixes the cut value), and top-k keeps ``x >= k-th largest`` with ``top_k`` as given."""
    if top_p is not None:
        srt = torch.sort(x, dim=-1)[0]
        remove = srt.softmax(-1).cumsum(-1) <= (1 - top_p)
        remove[..., -p_min_keep:] = False
        cut = srt.gather(-1, remove.sum(-1, keepdim=True))
        x = x.masked_fill(x < cut, -INF)
    if top_k is not None:
        kth = torch.topk(x, min(top_k, x.shape[-1]))[0][..., -1:]
        x = x.masked_fill(x < kth, -INF)
    return x


def rule_sample(logits, temps, procs, gen_rows, q, eos, ban):
    """sample_step with rule_filter: HF-style processor objects (top_k already folded) -> (ids [rows], the relative
    gap between the two largest p / q per row)."""
    x = apply_temperature(logits, torch.tensor(temps, dtype=torch.float32))
    top_p = p_keep = top_k = None
    greedy = 0
    for p in procs:
        if isinstance(p, CustomRepetitionPenaltyLogitsProcessorRepeat):
            x = repetition_penalty(gen_rows, x, p.penalty, p.max_input_ids, p.past_window)
        elif isinstance(p, TopPLogitsWarper):
            top_p, p_keep = p.top_p, p.min_tokens_to_keep
        elif isinstance(p, TopKLogitsWarper):
            top_k = p.top_k
        elif isinstance(p, ArgmaxOnly):
            greedy = 2 if p.exclude_eos else 1
    x = rule_filter(x, top_p, p_keep, top_k)
    if greedy:
        if greedy == 2:
            x[:, eos] = -INF
        x = x.masked_fill(x < x.max(dim=-1, keepdim=True)[0], -INF)
    if ban:
        x[:, eos] = -INF
    r = torch.softmax(x, -1) / q
    top2 = torch.topk(r, 2, dim=-1)[0]
    return sample_from_scores(torch.softmax(x, -1), q), (top2[:, 0] - top2[:, 1]) / top2[:, 0]


def _sp(procs, V):
    """SamplerParams of a processor tuple (gen_logits' shape: one min_keep for both warpers)."""
    sp = SamplerParams(top_p=None, top_k=None, repetition_penalty=1.0, penalty_max_ids=V - 1)
    for p in procs:
        if isinstance(p, CustomRepetitionPenaltyLogitsProcessorRepeat):
            sp.repetition_penalty, sp.penalty_max_ids, sp.penalty_window = p.penalty, p.max_input_ids, p.past_window
        elif isinstance(p, TopPLogitsWarper):
            sp.top_p, sp.min_keep = p.top_p, p.min_tokens_to_keep
        elif isinstance(p, TopKLogitsWarper):
            sp.top_k = p.top_k
        elif isinstance(p, ArgmaxOnly):
            sp.greedy, sp.greedy_exclude_eos = True, p.exclude_eos
    return sp


def _procs(tp, tk, rp, V):
    warp, proc = gen_logits(num_code=V - 1, top_P=tp, top_K=tk, repetition_penalty=rp)
    return (*proc, *warp)


def _signed_zero_rows(rows, V, g):
    """Negative logits, with 6 tokens at +0.0 and 6 at -0.0 in each row: 12 tokens tied at the maximum."""
    x = -(torch.rand(rows, V, generator=g) + 0.1)
    for r in range(rows):
        pos = torch.randperm(V, generator=g)[:12]
        x[r, pos[:6]] = 0.0
        x[r, pos[6:]] = -0.0
    return x


def _tie_rows(rows, V, g, ones):
    """``ones`` tokens at 1.0 and the rest at 0.0, positions shuffled per row (ones 0: a uniform row)."""
    x = torch.zeros(rows, V)
    for r in range(rows):
        x[r, torch.randperm(V, generator=g)[:ones]] = 1.0
    return x


def _edge(tag, rows, V, rpi, g):
    """(logits [rows, V] fp32, processors, temperatures, gen ids [rows / rpi, n_gen, rpi], eos, min_new, step,
    reference: 'oracle' or 'rule')."""
    randn = torch.randn(rows, V, generator=g)
    temps = [0.3, 0.5, 0.7, 1.0][:rpi]
    gen = torch.randint(0, 30, (rows // rpi, 23, rpi), generator=g)
    eos = V - 1
    d = dict(x=randn * 1.5, procs=_procs(0.7, 20, 1.05, V), temps=temps, gen=gen, min_new=0, step=0, ref="oracle")
    if tag == "temp_1e-3":
        d.update(temps=[1e-3] * rpi)
    elif tag == "temp_100":
        d.update(temps=[100.0] * rpi)
    elif tag == "logits_1e4":
        d.update(x=randn * 1e4, temps=[1.0] * rpi)
    elif tag == "underflow":  # three tokens 120 above the rest: every other probability is 0 in fp32
        x = randn * 1.5
        x[:, :3] += 120.0
        d.update(x=x, procs=_procs(None, None, 1.0, V), temps=[1.0] * rpi)
    elif tag == "neg_inf":
        x = (randn * 1.5).masked_fill(torch.rand(rows, V, generator=g) < 0.3, -INF)
        d.update(x=x)
    elif tag == "top_p_1":
        d.update(procs=_procs(1.0, None, 1.0, V))
    elif tag == "top_p_1e-6":
        d.update(procs=_procs(1e-6, None, 1.0, V))
    elif tag == "top_k_1":  # TopKLogitsWarper(1, min_tokens_to_keep=3): top_k 3
        d.update(procs=_procs(None, 1, 1.0, V))
    elif tag == "top_k_V-1":
        d.update(procs=_procs(None, V - 1, 1.0, V))
    elif tag == "top_k_ge_V":
        d.update(procs=_procs(None, V + 7, 1.0, V))
    elif tag == "ties_top_k":  # values on a grid of 0.5: the 20th largest is tied with its neighbours
        d.update(x=torch.round(randn * 3) / 2, procs=_procs(None, 20, 1.0, V))
    elif tag == "penalty_one_id_x31":  # a window of one id, 31 times: penalty_lut[31]; its logit < 0 in half the rows
        x = randn * 1.5
        wid = torch.randint(0, 30, (rows // rpi, rpi), generator=g)
        for r in range(rows):
            x[r, wid[r // rpi, r % rpi]] = -0.5 if r % 2 else 3.0
        d.update(x=x, gen=wid[:, None, :].expand(-1, 40, -1).contiguous(), procs=(
            CustomRepetitionPenaltyLogitsProcessorRepeat(1.3, V - 1, 31), *_procs(0.9, 40, 1.0, V)))
    elif tag == "penalty_rows_quirk":  # rows >= max_input_ids are not penalized (row index of the static batch)
        d.update(procs=(CustomRepetitionPenaltyLogitsProcessorRepeat(1.5, 2, 16), *_procs(0.7, 20, 1.0, V)),
                 gen=torch.randint(0, V, (rows // rpi, 23, rpi), generator=g))
    elif tag == "greedy_ties":
        d.update(x=torch.round(randn), procs=(*_procs(None, None, 1.0, V), ArgmaxOnly()))
    elif tag == "greedy_eos_max":
        x = randn * 1.5
        x[:, eos] = x.max(-1)[0] + 1.0
        d.update(x=x, procs=(*_procs(0.7, 20, 1.05, V), ArgmaxOnly(exclude_eos=True)), min_new=5, step=2)
    elif tag == "eos_ban_empty_row":  # only EOS is finite and it is banned: an all -inf row
        x = torch.full((rows, V), -INF)
        x[:, eos] = 1.0
        d.update(x=x, min_new=5, step=0)
    # the kernels' own rules (module docstring), against rule_sample
    elif tag == "rule_ties_top_p":  # 300 ones among 626 (HF's sort decides which 6 tied ones it removes)
        d.update(x=_tie_rows(rows, V, g, 300 * V // 626), procs=(TopPLogitsWarper(0.7, 3),), temps=[1.0] * rpi,
                 ref="rule")
    elif tag == "rule_ties_top_p_uniform":
        d.update(x=_tie_rows(rows, V, g, 0), procs=(TopPLogitsWarper(0.7, 3),), temps=[1.0] * rpi, ref="rule")
    elif tag == "rule_signed_zero_top_k":
        d.update(x=_signed_zero_rows(rows, V, g), procs=(TopKLogitsWarper(4),), temps=[1.0] * rpi, ref="rule")
    elif tag == "rule_signed_zero_greedy":
        d.update(x=_signed_zero_rows(rows, V, g), procs=(ArgmaxOnly(),), temps=[1.0] * rpi, ref="rule")
    elif tag == "rule_min_keep_p3_k1":  # HF: TopKLogitsWarper(1).top_k == 1, whatever top-p's min_tokens_to_keep
        d.update(x=randn * 0.3, procs=(TopPLogitsWarper(0.7, 3), TopKLogitsWarper(1)), temps=[1.0] * rpi, ref="rule")
    elif tag == "rule_min_keep_p5_k2":
        d.update(x=randn * 0.3, procs=(TopPLogitsWarper(0.05, 5), TopKLogitsWarper(2)), temps=[1.0] * rpi,
                 ref="rule")
    else:
        raise KeyError(tag)
    return d


C_ORACLE = ["temp_1e-3", "temp_100", "logits_1e4", "underflow", "neg_inf", "top_p_1", "top_p_1e-6", "top_k_1",
            "top_k_V-1", "top_k_ge_V", "ties_top_k", "penalty_one_id_x31", "penalty_rows_quirk", "greedy_ties",
            "greedy_eos_max", "eos_ban_empty_row"]
C_RULE = ["rule_ties_top_p", "rule_ties_top_p_uniform", "rule_signed_zero_top_k", "rule_signed_zero_greedy",
          "rule_min_keep_p3_k1", "rule_min_keep_p5_k2"]
PATHS = [(V_CODE, 4, 32), (V_TEXT, 1, 16)]  # (V, rows per item, rows): the sort path and the search path


@pytest.mark.parametrize("V,rpi,rows", PATHS, ids=["sort", "search"])
@pytest.mark.parametrize("tag", C_ORACLE + C_RULE)
def test_c_seeded_edges_exact(tag, V, rpi, rows):
    g = torch.Generator().manual_seed(zlib.crc32(tag.encode()) % 10000 + V)
    d = _edge(tag, rows, V, rpi, g)
    x, procs, temps, gen, eos = d["x"].float(), d["procs"], d["temps"], d["gen"], V - 1
    gen_rows = gen.permute(0, 2, 1).reshape(rows, -1)
    q = exp_noise(rows, V, 77)
    ban = d["step"] < d["min_new"]
    cfg = _cfg(procs, temps, eos, d["min_new"])
    out = sample_rows(x.cuda(), cfg, rpi, q.cuda(), gen.cuda(), step=d["step"]).cpu().long()
    assert bool(((out >= 0) & (out < V)).all())
    if d["ref"] == "oracle":
        sp = _sp(procs, V)
        ref = sample_step(x, gen_rows, torch.tensor(temps), sp, q, eos, ban)
        # margins per item: the repetition penalty reads each row's index within the batch
        margin = torch.tensor([min(decision_margins(x[i * rpi:(i + 1) * rpi], gen_rows[i * rpi:(i + 1) * rpi],
                                                    torch.tensor(temps), sp, q[i * rpi:(i + 1) * rpi], eos, ban))
                               for i in range(rows // rpi)]).repeat_interleave(rpi)
        if sp.penalty_max_ids < rows:  # decision_margins on one item would move the row >= max_input_ids cut
            margin = torch.full((rows,), INF)
    else:
        ref, margin = rule_sample(x, temps, procs, gen_rows, q, eos, ban)
    diff = torch.nonzero(out != ref)[:, 0].tolist()
    for r in diff:
        print(f"\nC {tag} V={V} row {r}: kernel {int(out[r])}, reference {int(ref[r])}, margin {float(margin[r]):.2e}")
        assert float(margin[r]) < MARGIN, (tag, V, r, int(out[r]), int(ref[r]), float(margin[r]))
    print(f"\nC {tag} V={V}: {rows - len(diff)} of {rows} ids equal, {len(diff)} margin exceptions")
    if tag == "eos_ban_empty_row":
        assert out.tolist() == [0] * rows


def test_c_rule_contains_the_oracle_kept_set():
    """rule_filter's top-p keeps a superset of the oracle's, larger only by tokens equal to the cut value; on rows
    without ties the two are the same set."""
    g = torch.Generator().manual_seed(5)
    for x in (_tie_rows(4, 626, g, 300), _tie_rows(4, 626, g, 0), torch.randn(4, 626, generator=g),
              _tie_rows(2, 21178, g, 10000)):
        orc = torch.isfinite(top_p_filter(x, 0.7, 3))
        rule_x = rule_filter(x, 0.7, 3, None)
        rule = torch.isfinite(rule_x)
        assert bool((orc <= rule).all())
        cut = rule_x.masked_fill(~rule, INF).min(-1, keepdim=True)[0]
        extra = rule & ~orc
        assert bool((x[extra] == cut.expand_as(x)[extra]).all())
        if len(torch.unique(x)) == x.numel():
            assert torch.equal(orc, rule)
    x = _tie_rows(1, 626, g, 300)
    print(f"\nC ties at the top-p cut, 300 ones / 326 zeros at top_p 0.7: oracle keeps "
          f"{int(torch.isfinite(top_p_filter(x, 0.7, 3)).sum())}, the kernels' rule "
          f"{int(torch.isfinite(rule_filter(x, 0.7, 3, None)).sum())}")


# the engine's k_sample<true> (prow = qi) against the float64 model, seeded, one request per edge configuration
ENGINE_EDGES = [("temp_1e-3", (0.7, 20, 1.05), [1e-3] * 4), ("temp_100", (0.7, 20, 1.05), [100.0] * 4),
                ("top_p_1", (1.0, None, 1.0), [0.7] * 4), ("top_p_1e-6", (1e-6, None, 1.0), [0.7] * 4),
                ("top_k_V-1", (None, V_CODE - 1, 1.0), [0.7] * 4), ("top_k_ge_V", (None, 1000, 1.0), [0.7] * 4),
                ("rows_quirk", "quirk", [0.5] * 4), ("min_keep_p3_k1", "mixed", [0.7] * 4)]


def _engine_procs(spec):
    """(processors, SamplerParams the float64 reference samples with)."""
    if spec == "quirk":  # penalty on codebooks 0 and 1 only: the engine's row index is the codebook
        return ((CustomRepetitionPenaltyLogitsProcessorRepeat(1.5, 2, 16), TopPLogitsWarper(0.7, 3),
                 TopKLogitsWarper(20, 3)), SamplerParams(top_p=0.7, top_k=20, repetition_penalty=1.5, penalty_max_ids=2))
    if spec == "mixed":  # top-k 1 after top-p keeps the maximum whatever top-p's min_keep: greedy over the row
        return ((TopPLogitsWarper(0.7, 3), TopKLogitsWarper(1)),
                SamplerParams(top_p=0.7, top_k=1, repetition_penalty=1.0, min_keep=1))
    tp, tk, rp = spec
    warp, proc = gen_logits(num_code=EOS, top_P=tp, top_K=tk, repetition_penalty=rp)
    return (*proc, *warp), SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp)


def test_c_engine_seeded_edges_against_float64():
    gpt, embed = sbd._gpt("plain", {}, 24, 2048)
    max_new = 160
    reqs, prompts, sps = [], [], []
    for i, (tag, spec, temps) in enumerate(ENGINE_EDGES):
        procs, sp = _engine_procs(spec)
        L = 10 + 3 * i
        p = synth_prompt_batch([L], seed=600 + i)[0][0]
        prompts.append(p)
        sps.append(sp)
        reqs.append(Request(emb=embed(p[None], torch.ones(1, L, dtype=torch.bool))[0], temperature=temps,
                            eos_token=EOS, max_new_token=max_new, min_new_token=max_new, logits_processors=procs,
                            manual_seed=700 + i))
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 4, max_new, False, 0)
        for i, slot, n in schedule(reqs, dev, 64):
            got[i] = dev.harvest(slot, n).ids[0].cpu().clone()
    orc = _f64()
    for i, (tag, spec, temps) in enumerate(ENGINE_EDGES):
        ids = got[i]
        assert ids.shape == (max_new, 4), (tag, ids.shape)
        _, lg = orc.teacher_forced(orc.embed_prompt(prompts[i]), ids)
        sampled, margins = sample_trace(lg, ids, torch.tensor(temps), sps[i], exp_noise(4, V_CODE, 700 + i), EOS,
                                        max_new)
        exc = 0
        for t in range(max_new):
            if not torch.equal(sampled[t], ids[t].long()):
                print(f"\nC engine {tag} step {t}: {ids[t].tolist()} vs {sampled[t].tolist()}, "
                      f"margin {float(margins[t]):.2e}")
                assert margins[t] < MARGIN, (tag, t, ids[t].tolist(), sampled[t].tolist(), float(margins[t]))
                exc += 1
        print(f"\nC engine {tag}: {max_new - exc} of {max_new} steps equal, {exc} margin exceptions")


# k_flow's in-kernel sampler against k_sample (two handles over one blob), on the edge configurations a model's
# logits can reach
FLOW_EDGES = [("temp_1e-3", sbd._procs((0.7, 20, 1.05)), [1e-3] * 4),
              ("temp_100", sbd._procs((0.7, 20, 1.05)), [100.0] * 4),
              ("top_p_1", (TopPLogitsWarper(1.0, 3),), [0.7] * 4),
              ("top_p_1e-6", (TopPLogitsWarper(1e-6, 3),), [0.7] * 4),
              ("top_k_1", (TopKLogitsWarper(1, 3),), [0.7] * 4),
              ("top_k_V-1", (TopKLogitsWarper(V_CODE - 1, 3),), [0.7] * 4),
              ("top_k_ge_V", (TopKLogitsWarper(1000, 3),), [0.7] * 4),
              ("min_keep_p3_k1", (TopPLogitsWarper(0.7, 3), TopKLogitsWarper(1)), [0.7] * 4),
              ("rows_quirk", (CustomRepetitionPenaltyLogitsProcessorRepeat(1.5, 2, 16), TopPLogitsWarper(0.7, 3)),
               [0.5] * 4)]


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("case", FLOW_EDGES, ids=[c[0] for c in FLOW_EDGES])
def test_c_flow_in_kernel_sampler_edges(case, B, monkeypatch):
    tag, procs, temps = case
    outs = sbd._both(f"C flow {tag} B={B}", B, monkeypatch, procs=procs, temp=temps, min_new=200, max_new=200,
                     seed=55)
    print(f"\nC flow {tag} B={B}: identical over {int(outs[-1].ids[0].shape[0])} steps")
