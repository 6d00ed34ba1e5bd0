"""The float64 reference of tests/f64_oracle.py on the CPU: it is the fp32 oracle's model (and its fp16 variant the
fp16 oracle's), its single teacher-forced pass is the step-by-step decode loop, and the peaked-attention model of
tests/test_gpu_long_attention.py is as peaked as that file says while its fp16 cache stays far from overflow."""
import torch

from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from f64_oracle import F64Oracle, peaked_state, sample_trace, top_k_margin
from fp16_oracle import GPTOracleFp16
from oracle.gpt_oracle import GPTOracle, SamplerParams, exp_noise

MARGIN = 1e-3
TEMP = torch.tensor([0.3, 0.5, 0.7, 1.0])


def _cut(gs, layers=4):
    """The first ``layers`` layers of the synthetic model (the step-by-step oracles' cost is per layer)."""
    return {k: v for k, v in gs.items() if not k.startswith("layers.") or int(k.split(".")[1]) < layers}


def _oracle_run(orc, length=21, steps=12, seed=11, pseed=4):
    ids, mask, tmask = synth_prompt_batch([length], seed=pseed)
    out = orc.generate(orc.embed_prompt(ids, tmask), ids, TEMP, 625, attention_mask=mask, max_new_token=steps,
                       min_new_token=steps, sampler=SamplerParams(), return_hidden=True, manual_seed=seed, trace=True)
    return ids[0], out


def _compare(orc, ref, atol):
    prompt, out = _oracle_run(orc)
    ids, hid = out.ids[0], out.hiddens[0]
    h64, lg = ref.teacher_forced(ref.embed_prompt(prompt), ids)
    err = float((h64 - hid.double()).abs().max())
    assert err < atol, err
    sampled, margins = sample_trace(lg, ids, TEMP, SamplerParams(), exp_noise(4, 626, 11), 625, ids.shape[0])
    flips = [i for i in range(ids.shape[0]) if not torch.equal(sampled[i], ids[i])]
    assert all(margins[i] < MARGIN for i in flips), (flips, margins)
    assert len(flips) <= 1, flips
    return err, len(flips)


def test_f64_follows_the_fp32_oracle():
    gs, es = _cut(synth_gpt_state(0)), synth_embed_state(1)
    err, flips = _compare(GPTOracle(gs, es), F64Oracle(gs, es), 1e-5)
    print(f"\n|f64 - fp32 oracle| = {err:.2e}, margin-accepted ids {flips}")


def test_fp16_variant_follows_the_fp16_oracle():
    """The fp16 oracle rounds an fp32 K/V to fp16, this one a float64 K/V: now and then the two round an element to
    neighbouring fp16 values (one fp16 ulp, ~5e-4 relative), which moves the hidden states by ~2e-5 on this four-layer
    cut (~2e-4 on all 20 layers)."""
    gs, es = _cut(synth_gpt_state(0)), synth_embed_state(1)
    for layers, kv in ((True, True), (False, True)):
        err, flips = _compare(GPTOracleFp16(gs, es, fp16_layers=layers, fp16_kv=kv),
                              F64Oracle(gs, es, fp16_layers=layers, fp16_kv=kv), 2e-4)
        print(f"\nfp16 layers={layers} kv={kv}: |f64 - fp16 oracle| = {err:.2e}, margin-accepted ids {flips}")


def test_fp16_variant_rounds_k_and_v():
    gs, es = synth_gpt_state(0), synth_embed_state(1)
    prompt = synth_prompt_batch([9], seed=4)[0][0]
    for kv in (True, False):
        ref = F64Oracle(gs, es, fp16_layers=True, fp16_kv=kv)
        _, qkvs = ref.forward(ref.embed_prompt(prompt), return_qkv=True)
        assert all(torch.equal(t, t.half().double()) for _, k, v in qkvs for t in (k, v)) == kv


def peaked_stats(T_codes=1024, seed=3):
    """Attention statistics of the peaked model over a 16-token text prompt and ``T_codes`` random code frames, fp32:
    (per layer: score std over the last 64 queries' causal scores, median spread max - min of a query's scores), and
    the largest |K| and |V| any layer caches."""
    gs, es = synth_gpt_state(0), synth_embed_state(1)
    ref = F64Oracle(peaked_state(gs), es, dtype=torch.float32)
    g = torch.Generator().manual_seed(seed)
    x = torch.cat([ref.embed_prompt(torch.randint(1, 1000, (16,), generator=g)),
                   ref.embed_codes(torch.randint(0, 625, (T_codes, 4), generator=g))])
    T = x.shape[0]
    _, qkvs = ref.forward(x, return_qkv=True)
    stds, spreads = [], []
    for q, k, _ in qkvs:
        sc = torch.matmul(q[:, -64:], k.transpose(1, 2)) * 64 ** -0.5  # [H, 64, T]
        sc = sc[:, :, : T - 64]  # keys every one of the 64 queries sees
        stds.append(float(sc.std()))
        spreads.append(float((sc.max(-1).values - sc.min(-1).values).median()))
    kmax = max(float(k.abs().max()) for _, k, _ in qkvs)
    vmax = max(float(v.abs().max()) for _, _, v in qkvs)
    return stds, spreads, kmax, vmax


def test_peaked_model_scores_and_fp16_range():
    """The peaked model (q_proj and k_proj x 4) at a ~1000-key context: scores have a std of several units in every
    layer (the synthetic model's ~0.3, x 16) and a query's scores spread over tens, while the largest |K| the fp16
    cache holds stays three orders of magnitude below fp16's 65504."""
    stds, spreads, kmax, vmax = peaked_stats()
    print(f"\npeaked model: score std per layer {min(stds):.1f}..{max(stds):.1f}, median spread "
          f"{min(spreads):.0f}..{max(spreads):.0f}, max |K| {kmax:.1f}, max |V| {vmax:.2f}")
    assert kmax < 65.504 and vmax < 65.504
    assert min(stds) > 2.5 and min(spreads) > 15


def test_top_k_margin_is_the_gap_at_the_cut():
    logits = torch.tensor([[5.0, 4.0, 3.0, 2.5, 2.4999, 0.0]], dtype=torch.float64)
    sp = SamplerParams(top_p=None, top_k=4, repetition_penalty=1.0)
    assert abs(top_k_margin(logits, torch.zeros(1, 0, dtype=torch.long), torch.tensor([1.0]), sp) - 1e-4) < 1e-9
    sp = SamplerParams(top_p=None, top_k=None, repetition_penalty=1.0)
    assert top_k_margin(logits, torch.zeros(1, 0, dtype=torch.long), torch.tensor([1.0]), sp) == float("inf")


def test_text_rows_follow_the_fp32_oracle():
    """teacher_forced_text is the oracle's infer_text loop: text ids fed back through emb_text, the text head's logits
    sampled with the text request's noise."""
    gs, es = _cut(synth_gpt_state(0)), synth_embed_state(1)
    orc, ref = GPTOracle(gs, es), F64Oracle(gs, es)
    ids, mask, tmask = synth_prompt_batch([13], seed=6)
    steps, temp, sp = 10, torch.tensor([0.7]), SamplerParams(penalty_max_ids=21177)
    out = orc.generate(orc.embed_prompt(ids, tmask), ids, temp, 21001, attention_mask=mask, max_new_token=steps,
                       min_new_token=steps, sampler=sp, infer_text=True, return_hidden=True, manual_seed=5)
    got, hid = out.ids[0], out.hiddens[0]
    assert got.shape == (steps,)
    h64, lg = ref.teacher_forced_text(ref.embed_prompt(ids[0]), got)
    assert lg.shape == (steps, 1, 21178)
    err = float((h64 - hid.double()).abs().max())
    assert err < 1e-5, err
    sampled, margins = sample_trace(lg, got[:, None], temp, sp, exp_noise(1, 21178, 5), 21001, steps)
    flips = [i for i in range(steps) if int(sampled[i, 0]) != int(got[i])]
    assert all(margins[i] < MARGIN for i in flips) and len(flips) <= 1, (flips, margins)
