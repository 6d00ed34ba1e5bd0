"""Refined split-text paragraphs without a GPU: the stage graph's join (``core._RefineGraph``) in the scheduling policy
against a stub device, a ``ChatEngine`` on a stub device and a stand-in ``Chat`` (failures, cancels in every phase,
nothing left held), and ``Request.noise_batch``: its rows and its validation."""
import time
from types import SimpleNamespace

import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.core import Chat, ChatEngine, _RefineGraph
from chattts_b200.engine import Arrivals, Request, ScheduleStats, _poll_cycles, check_noise_batch, noise_rows
from chattts_b200.processors import exp_noise, gen_logits
from test_online_cpu import OnlineStub, _drain, _req


# ---------------------------------------------------------------------------------------------------- the join
def _graph(n, ref_len, code_len=5, reference=True):
    made = []  # (sentence, text, sample, request) in the order the code requests were made

    def code(k, text, sample):
        r = _req(code_len, seed=100 + k)
        made.append((k, text, sample, r))
        return r

    g = _RefineGraph(n, lambda out: f"r{int(out.ids[0].shape[0])}", code,
                     (lambda text: _req(ref_len, seed=99)) if reference else None,
                     (lambda ref: "spk") if reference else None)
    return g, made


def _refinements(g, lengths):
    return [_req(n, seed=k, then=g.then(k), text=True) for k, n in enumerate(lengths)]


def _origin(requests, stats, made):
    """sentence -> ("fanout", position) or ("child", parent request index) of its code request."""
    where = {}
    for k, _, _, r in made:
        i = next(j for j in range(len(requests)) if requests[j] is r)
        for p, kids in stats.fanout.items():
            if i in kids:
                where[k] = ("fanout", kids.index(i))
        for p, c in stats.children.items():
            if c == i:
                where[k] = ("child", p)
    return where


def test_join_before_at_and_after_the_reference_stage():
    """Four slots, chunk 8: refinements 0 and 1 end at the first poll (1 waits for the sample), the reference stage
    (17 tokens) ends with refinement 2 (25 tokens, in a higher slot: the reference's then runs first), refinement 3
    (41 tokens) ends after it."""
    requests, src = [], Arrivals()
    g, made = _graph(4, ref_len=17)
    src.submit(_refinements(g, [9, 9, 25, 41]), key="paragraph")
    dev = OnlineStub(4, requests)
    stats = ScheduleStats()
    gen = _poll_cycles(requests, dev, 8, stats=stats, source=src)
    _drain(gen, src)
    assert sorted(k for k, *_ in made) == [0, 1, 2, 3]  # each exactly once (the graph asserts it as well)
    assert [k for k, *_ in made] == [0, 1, 2, 3]
    where = _origin(requests, stats, made)
    assert where[0] == ("fanout", 0) and where[1] == ("fanout", 1)  # refined before the sample: the fan-out, in order
    assert where[2] == ("child", 2) and where[3] == ("child", 3)  # refined once the sample was known
    assert stats.children[0] == 4 and requests[4] is g.ref  # refinement 0's follow-up is the reference stage
    assert g.refined == ["r9", "r9", "r25", "r41"]
    assert all(s == ("spk", "r9") for _, _, s, _ in made)


def test_join_when_a_refinement_s_then_runs_first_at_the_reference_poll():
    """Fillers hold slots 0 and 1 until refinements 1 and 2 take them; refinement 0 sits in slot 2, so the reference
    stage lands there, above refinement 2, which ends at the same poll and whose then therefore runs first."""
    requests, src = [], Arrivals()
    g, made = _graph(3, ref_len=17)
    src.submit(_req(9))
    src.submit(_req(9))
    src.submit(_refinements(g, [17, 100, 25]), key="paragraph")
    dev = OnlineStub(3, requests)
    stats = ScheduleStats()
    gen = _poll_cycles(requests, dev, 8, stats=stats, source=src)
    _drain(gen, src)
    ref_slot = next(s for batch in dev.admissions for s, i in batch if requests[i] is g.ref)
    r2_slot = next(s for batch in dev.admissions for s, i in batch if i == 4)
    assert r2_slot < ref_slot
    where = _origin(requests, stats, made)
    assert where == {0: ("fanout", 0), 2: ("fanout", 1), 1: ("child", 3)}
    assert [k for k, *_ in made] == [0, 2, 1]


@pytest.mark.parametrize("n", [1, 3])
def test_without_a_reference_stage_each_refinement_makes_its_code_request(n):
    requests, src = [], Arrivals()
    g, made = _graph(n, ref_len=17, reference=False)
    src.submit(_refinements(g, [9, 25, 17][:n]), key="paragraph")
    dev = OnlineStub(4, requests)
    stats = ScheduleStats()
    _drain(_poll_cycles(requests, dev, 8, stats=stats, source=src), src)
    assert g.ref is None and not stats.fanout
    assert {k: c for k, c in _origin(requests, stats, made).items()} == {k: ("child", k) for k in range(n)}
    assert all(s is None for _, _, s, _ in made)


def test_the_graph_refuses_an_empty_refinement():
    g, made = _graph(2, ref_len=17)
    empty = SimpleNamespace(ids=[torch.zeros(0, dtype=torch.long)])
    with pytest.raises(RuntimeError, match="ended empty"):
        g.then(1)(empty)
    assert g.refined == [None, None] and not made


# ---------------------------------------------------------------------------------------------------- ChatEngine
class _FakeChat:
    """The parts of ``Chat`` a ``ChatEngine`` paragraph touches.  Sentence t's refinement yields ``refine_len[t]``
    tokens (0: EOS first) and is the text 'R' + t; the code request of 'R' + t (or of t) yields ``code_len[t]``."""

    def __init__(self, refine_len, code_len, max_batch=4):
        self.refine_len, self.code_len = refine_len, code_len
        self.gpt = SimpleNamespace(max_batch=max_batch)
        self.speaker = SimpleNamespace(encode_prompt=lambda codes: "spk")
        self.dvae = SimpleNamespace(audio_encoder=SimpleNamespace(encode_rows=lambda wavs: [None] * len(wavs)),
                                    engine=SimpleNamespace(decode_rows=lambda rows, k: [
                                        torch.ones(512 * int(r.shape[0])) for r in rows]))
        self.decoder = self.dvae
        self.codes = []  # (text, params, request) of every code request, in the order they were made
        self.texts = {}  # refinement request -> its sentence

    def normalizer(self, text, *args):
        return text

    def _refine_request(self, text, params, noise_batch=None):
        r = Request(emb=torch.zeros(3, 4), temperature=[0.7], eos_token=1, max_new_token=params.max_new_token,
                    manual_seed=params.manual_seed, infer_text=True, noise_batch=noise_batch)
        self.texts[r] = text
        return r

    def _code_request(self, text, params, noise_batch=None):
        r = Request(emb=torch.zeros(3, 4), temperature=[0.3] * 4, eos_token=625, max_new_token=params.max_new_token,
                    manual_seed=params.manual_seed, noise_batch=noise_batch)
        self.codes.append((text, params, r))
        return r

    def _refined_text(self, out):
        return "R" + out.text

    def length(self, r):
        if r in self.texts:
            return self.refine_len[self.texts[r]]
        text = next(t for t, _, c in self.codes if c is r)
        return self.code_len[text[1:] if text[1:] in self.code_len else text]


class _Stub(OnlineStub):
    """OnlineStub with the engine's id buffer (the window decode reads it), an admission hook, and harvests that name
    the sentence of the refinement they come from."""

    def __init__(self, slots, requests, chat, on_admit):
        super().__init__(slots, requests)
        self.ids_out = torch.zeros(slots, 256, 4, dtype=torch.int32)
        self.chat, self.on_admit, self.owner = chat, on_admit, {}

        class Lengths:
            def __getitem__(_, i):
                return chat.length(requests[i])

        self.lengths = Lengths()

    def admit(self, batch):
        for s, i in batch:
            self.owner[s] = self.requests[i]
        super().admit(batch)
        for _, i in batch:
            self.on_admit(self.requests[i])

    def harvest(self, slot, n, copy=True):
        out = super().harvest(slot, n, copy)
        out.text = self.chat.texts.get(self.owner[slot])
        return out

    def empty(self, index=None):
        out = super().empty(index)
        out.text = self.chat.texts.get(self.requests[index])
        return out


def _open(chat, slots=4, on_admit=lambda r: None):
    devs = []

    def make(requests):
        devs.append(_Stub(slots, requests, chat, on_admit))
        return devs[-1]

    eng = ChatEngine(make, 8, None, None, None, chat, False, max_new_cap=200)
    return eng, devs


PARA = "a. b. c. d. e"
SENTENCES = ["a. ", "b. ", "c. ", "d. ", "e"]


def _chat(refine=(9, 9, 25, 41, 17), code=(9, 17, 25, 9, 33), **kw):
    return _FakeChat(dict(zip(SENTENCES, refine)), dict(zip(SENTENCES, code)), **kw)


def _params(**kw):
    return (Chat.InferCodeParams(manual_seed=3, max_new_token=200, **kw),
            Chat.RefineTextParams(manual_seed=5, max_new_token=200))


def _idle(devs):
    return all(st != _lib.SLOT_RUNNING for d in devs for st in d.state)


@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_chat_engine_runs_a_refined_paragraph_s_stage_graph(m):
    chat = _chat()
    p, r = _params()
    eng, devs = _open(chat)
    with eng:
        job = eng.submit(PARA, params_infer_code=p, split_text=True, skip_refine_text=False, params_refine_text=r,
                         max_split_batch=m)
        wav = job.result(timeout=30)
    assert job.refined == ["R" + s for s in SENTENCES] and job.spk_smp == "spk"
    (ref_text, ref_params, ref), *codes = chat.codes
    assert ref_text == "Ra. " and ref.noise_batch is None and ref_params is not p  # reference: a batch of one
    assert sorted(t for t, _, _ in codes) == sorted(job.refined)
    n = len(SENTENCES)
    for t, q, c in codes:
        k = job.refined.index(t)
        assert c.noise_batch == (min(m, n - m * (k // m)), k % m)
        assert (q.spk_smp, q.txt_smp) == ("spk", "Ra. ") and q is not p
    assert p.spk_smp is None and p.txt_smp is None  # the caller's params are not modified
    assert [x.noise_batch for x in chat.texts] == [(4, 0), (4, 1), (4, 2), (4, 3), (1, 0)]  # rows of max_batch 4
    assert wav.shape == (sum(512 * chat.code_len[s] - 256 for s in SENTENCES),)
    assert eng._requests.held() == 0 and not eng._pending and _idle(devs)


def test_an_explicit_spk_smp_or_one_sentence_skips_the_reference_stage():
    chat = _chat()
    chat.refine_len["just one"] = chat.code_len["just one"] = 9
    p, r = _params(spk_smp="given")
    eng, _ = _open(chat)
    with eng:
        job = eng.submit(PARA, params_infer_code=p, split_text=True, skip_refine_text=False, params_refine_text=r)
        job.result(timeout=30)
        assert len(chat.codes) == len(SENTENCES) and job.spk_smp is None
        assert all(q.spk_smp == "given" for _, q, _ in chat.codes)
        chat.codes.clear()
        one = eng.submit("just one", params_infer_code=_params()[0], split_text=True, skip_refine_text=False,
                         params_refine_text=r)
        one.result(timeout=30)
    assert [t for t, _, _ in chat.codes] == ["Rjust one"] and one.refined == ["Rjust one"]
    assert eng._requests.held() == 0


@pytest.mark.parametrize("case", ["empty refinement", "reference too short"])
def test_a_failing_stage_fails_the_job_and_cancels_its_other_stages(case):
    # sentence 2's refinement ends empty at the first poll, or the reference stage (1 token) cannot be encoded; either
    # way sentences 3 and 4 are still refining (150 tokens) and are cancelled at the next poll
    chat = _chat(refine=(9, 9, 0 if case == "empty refinement" else 9, 150, 150),
                 code=(1 if case == "reference too short" else 9, 9, 9, 9, 9))
    p, r = _params()
    eng, devs = _open(chat)
    with eng:
        job = eng.submit(PARA, params_infer_code=p, split_text=True, skip_refine_text=False, params_refine_text=r)
        other = eng.submit("x. y", params_infer_code=_params()[0], split_text=True)  # an unrelated job goes on
        chat.code_len.update({"x. ": 40, "y": 40})
        with pytest.raises((RuntimeError, _lib.CtbError)):
            job.result(timeout=30)
        other.result(timeout=30)
    assert devs[0].cancels  # the running refinements were stopped, not run to their 150 tokens
    assert max(n for d in devs for n in d.done) < 150
    assert eng._requests.held() == 0 and not eng._pending and _idle(devs)


@pytest.mark.parametrize("phase", ["waiting", "refinement", "reference", "code"])
def test_a_cancel_in_every_phase_leaves_nothing_held(phase):
    chat = _chat(refine=(9, 9, 25, 41, 17), code=(17, 40, 40, 40, 40))
    chat.refine_len.update({"x. ": 9, "y": 9})
    chat.code_len.update({"x. ": 17, "y": 17})
    held = {}

    def on_admit(r):
        job = held.get("job")
        if job is None or held.get("done"):
            return
        if r.infer_text:
            mine, stage = chat.texts[r] in SENTENCES, "refinement"
        else:  # the paragraph's reference stage is the one code request of it without a noise_batch
            text = next(t for t, _, c in chat.codes if c is r)
            mine, stage = text[1:] in SENTENCES, "reference" if r.noise_batch is None else "code"
        if mine and stage == phase:
            held["done"] = True
            job.cancel()

    eng, devs = _open(chat, on_admit=on_admit)
    with eng:
        with eng._source._cv:  # the worker takes both submissions (and a waiting cancel) at one poll
            job = eng.submit(PARA, params_infer_code=_params()[0], split_text=True, skip_refine_text=False,
                             params_refine_text=_params()[1])
            other = eng.submit("x. y", params_infer_code=_params()[0], split_text=True, skip_refine_text=False,
                               params_refine_text=_params()[1])
            held["job"] = job
            if phase == "waiting":
                held["done"] = True
                job.cancel()
        wav = other.result(timeout=30)
    assert held.get("done") and job.cancelled() and job.done()
    assert wav.shape == (2 * (512 * 17 - 256),)
    assert eng._requests.held() == 0 and not eng._pending and not eng._job_at and _idle(devs)


def test_max_split_batch_over_max_batch_is_refused_at_submit():
    chat = _chat(max_batch=4)
    eng, _ = _open(chat)
    with eng:
        p, r = _params()
        with pytest.raises(ValueError, match="max_batch"):
            eng.submit(PARA, params_infer_code=p, split_text=True, max_split_batch=5)
        with pytest.raises(ValueError, match="max_split_batch"):
            eng.submit(PARA, params_infer_code=p, split_text=True, max_split_batch=0)
        eng.submit("a. b", params_infer_code=p, split_text=True, max_split_batch=5, skip_refine_text=False,
                   params_refine_text=r).cancel()  # two sentences: a batch of 2


# ---------------------------------------------------------------------------------------------------- Chat's driver
class _DriverStub(_Stub):
    """_Stub that records each decode's chunk and calls ``on_decode(number of decodes so far)`` after each one.  The
    hidden path reads the id buffer (the stand-in decoders only count tokens)."""

    def __init__(self, slots, requests, chat, on_admit, on_decode):
        super().__init__(slots, requests, chat, on_admit)
        self.on_decode, self.chunks, self.hid_out = on_decode, [], self.ids_out

    def decode(self, n):
        self.chunks.append(n)
        super().decode(n)
        self.on_decode(self.decodes)


@pytest.fixture
def driver(monkeypatch):
    """``make(fake, ...)``: a real ``Chat`` whose models are the ``_FakeChat``'s and whose GPT handle serves its
    engines on ``_DriverStub`` devices, so ``infer_continuous*`` runs its own driver unchanged."""
    import ctypes as C

    import chattts_b200.engine as engine
    from chattts_b200.gpt import GPT

    made = []

    def make(fake, max_batch=4, on_admit=lambda r: None, on_decode=lambda c, k: None, stub=_DriverStub):
        c = Chat()
        c.gpt = GPT({"hidden_size": 4}, embed=None, device_gpt=torch.device("cpu"), max_batch=max_batch,
                    max_context=300)
        c.gpt._handle = C.c_void_p(1)  # never reaches the library: the device layer is a stub
        made.append(c.gpt)
        c.vocos = c.embed = c.tokenizer = c.device = None
        c.decoder = c.dvae = fake.dvae
        c.speaker, c.normalizer = fake.speaker, fake.normalizer
        c._code_request, c._refine_request, c._refined_text = fake._code_request, fake._refine_request, \
            fake._refined_text
        devs = []

        def device(gpt, requests, S, cap, hidden):
            devs.append(stub(S, requests, fake, on_admit, lambda k: on_decode(c, k)))
            return devs[-1]

        monkeypatch.setattr(engine, "EngineDevice", device)
        return c, devs

    yield make
    for gpt in made:
        gpt._handle = C.c_void_p()


TEXTS = ["t0", "t1", "t2", "t3", "t4", "t5"]


def _text_chat(code=150, refine=9, **kw):
    return _FakeChat({t: refine for t in TEXTS}, {t: code for t in TEXTS}, **kw)


@pytest.mark.parametrize("n", [3, 6])
@pytest.mark.parametrize("split_text", [False, True])
def test_the_first_admission_holds_a_first_stage_of_every_text_it_can(driver, n, split_text):
    fake = _text_chat()
    texts = TEXTS[:n]
    if split_text:  # two sentences each: a paragraph's first stage is its reference stage
        texts = [t + ". x" for t in texts]
        fake.code_len.update({t: 20 for t in ["x", *(t + ". " for t in TEXTS)]})
    c, devs = driver(fake)
    p = Chat.InferCodeParams(manual_seed=1, max_new_token=200)
    got = dict(c.infer_continuous(texts, params_infer_code=p, split_text=split_text))
    assert sorted(got) == list(range(n))
    assert len(devs[0].admissions[0]) == min(4, n)  # every slot the call has, or one per text


@pytest.mark.parametrize("case", ["plain", "stream", "one text", "split", "split stream", "env"])
def test_default_slots_and_poll_interval(driver, monkeypatch, case):
    fake = _text_chat(code=20)
    fake.code_len.update({"x": 20, "y": 20})
    c, devs = driver(fake)
    texts, split = (TEXTS[:1] if case == "one text" else TEXTS[:3]), case.startswith("split")
    if split:
        texts = ["x"] * 3  # one sentence each
    if case == "env":
        monkeypatch.setenv("CTB_DECODE_CHUNK", "5")
    else:
        monkeypatch.delenv("CTB_DECODE_CHUNK", raising=False)
    params = [Chat.InferCodeParams(manual_seed=1, max_new_token=200, stream_batch=b) for b in (16, 12, 20)][:len(texts)]
    if case.endswith("stream"):
        list(c.infer_continuous_stream(texts, params_infer_code=params, split_text=split))
    else:
        list(c.infer_continuous(texts, params_infer_code=params, split_text=split))
    want_slots = {"one text": 2, "split": 4, "split stream": 4}.get(case, 3)
    want_chunk = {"stream": 12, "split": 24, "split stream": 24, "env": 5}.get(case, 32)
    assert devs[0].slots == want_slots and set(devs[0].chunks) == {want_chunk}


@pytest.mark.parametrize("stream", [False, True])
def test_an_interrupt_ends_the_running_texts_with_what_they_have(driver, caplog, stream):
    fake = _text_chat(code=150)

    def on_decode(c, k):
        if k == 2:
            c.interrupt()

    c, devs = driver(fake, on_decode=on_decode)
    p = Chat.InferCodeParams(manual_seed=1, max_new_token=200, stream_speed=3000, pass_first_n_batches=0)
    call = c.infer_continuous_stream if stream else c.infer_continuous
    with caplog.at_level("WARNING"):
        events = list(call(TEXTS[:4], params_infer_code=p, slots=2))
    assert "generation is interrupted" in caplog.text
    partial = 512 * (1 + 2 * (24 if stream else 32)) - 256  # the prefill's token and two polls' chunks
    if stream:
        finals = [(i, x) for i, x, last in events if last]
        assert sorted(i for i, _ in finals) == [0, 1] and {i for i, *_ in events} == {0, 1}
        assert all(sum(x.shape[1] for j, x, _ in events if j == i) == partial for i in (0, 1))
    else:
        assert sorted(i for i, _ in events) == [0, 1] and all(w.shape == (partial,) for _, w in events)
    assert c.gpt._open is None and len(devs[0].chunks) == 2  # the handle is free, and nothing decoded after the read


def test_batched_refinement_speaks_the_refined_texts_as_they_are(driver):
    fake = _text_chat(code=20)
    fake.normalizer = lambda text, *a: "N:" + text  # not the identity, so a second pass would show
    c, _ = driver(fake)
    refined_in = []

    def refine_text(texts, device, params):  # batch b's row k refines to ids [100 b + k]
        refined_in.append(list(texts))
        return SimpleNamespace(ids=[torch.tensor([100 * len(refined_in) + k]) for k in range(len(texts))],
                               destroy=lambda: None)

    c._refine_text = refine_text
    c.tokenizer = SimpleNamespace(break_0_ids=10 ** 6, decode=lambda tokens: [f"r{int(t[0])}" for t in tokens])
    want = ["r100", "r101", "r102", "r103", "r200", "r201"]
    fake.code_len.update({t: 20 for t in want})
    p = Chat.InferCodeParams(manual_seed=1, max_new_token=200)
    got = dict(c.infer_continuous(TEXTS, params_infer_code=p, skip_refine_text=False,
                                  params_refine_text=Chat.RefineTextParams(manual_seed=2)))
    assert sorted(got) == list(range(6))
    assert refined_in == [["N:" + t for t in TEXTS[:4]], ["N:" + t for t in TEXTS[4:]]]  # batches of max_batch
    assert [t for t, _, _ in fake.codes] == want


@pytest.mark.parametrize("stream", [False, True])
def test_a_text_whose_refinement_ends_empty_speaks_the_empty_refinement(driver, stream):
    fake = _text_chat(code=20, refine=0)  # seeded: every refinement samples EOS first
    fake.code_len.update({"R" + t: 20 for t in TEXTS})
    c, _ = driver(fake)
    p = Chat.InferCodeParams(manual_seed=1, max_new_token=200)
    kw = dict(params_infer_code=p, skip_refine_text=False, refine_on_engine=True,
              params_refine_text=Chat.RefineTextParams(manual_seed=2, max_new_token=50))
    if stream:
        got = {i for i, _, last in c.infer_continuous_stream(TEXTS[:2], **kw) if last}
    else:
        got = {i for i, w in c.infer_continuous(TEXTS[:2], **kw) if w.shape == (512 * 20 - 256,)}
    assert got == {0, 1} and [t for t, _, _ in fake.codes] == ["Rt0", "Rt1"]


class _SlowStub(_DriverStub):
    def decode(self, n):
        time.sleep(0.02)  # a poll takes longer than the driver's wait for the next chunk
        super().decode(n)


@pytest.mark.parametrize("stream", [False, True])
def test_an_interrupt_cancels_every_unfinished_paragraph(driver, caplog, stream):
    # the reference stages and sentence 0 end in one poll of 24 steps each: sentence 0's chunks are out before the
    # interrupt, while the other sentences need 7 polls
    fake = _chat(code=(9, 150, 150, 150, 150))

    def on_decode(c, k):
        if k == 3:
            c.interrupt()

    c, devs = driver(fake, on_decode=on_decode, stub=_SlowStub)
    p = Chat.InferCodeParams(manual_seed=1, max_new_token=200)
    call = c.infer_continuous_stream if stream else c.infer_continuous
    with caplog.at_level("WARNING"):
        events = list(call([PARA, PARA], params_infer_code=p, split_text=True))
    assert "generation is interrupted" in caplog.text
    if stream:
        assert events and not any(last for *_, last in events)
    else:
        assert events == []
    assert max(d.decodes for d in devs) < 3 + 6 and c.gpt._open is None and _idle(devs)


# ---------------------------------------------------------------------------------------------------- noise_batch
def _nreq(noise_batch=None, seed=7, text=False, penalty=None):
    procs = ()
    if penalty is not None:
        _, procs = gen_logits(num_code=penalty, top_P=None, top_K=None, repetition_penalty=1.05)
    return Request(emb=torch.zeros(3, 4), temperature=[0.7] if text else [0.3] * 4, eos_token=1, manual_seed=seed,
                   infer_text=text, noise_batch=noise_batch, logits_processors=tuple(procs))


@pytest.mark.parametrize("rows", [1, 4])
def test_noise_rows_are_slices_of_the_static_batch_s_noise(rows):
    cols = 37
    reqs = [_nreq((3, 0)), _nreq((3, 2)), _nreq(None), _nreq((1, 0)), _nreq((5, 4), seed=9), _nreq((3, 1), seed=8)]
    cache = {}
    got = noise_rows(reqs, rows, cols, cache)
    want = torch.cat([exp_noise(3 * rows, cols, 7)[0: rows], exp_noise(3 * rows, cols, 7)[2 * rows: 3 * rows],
                      exp_noise(rows, cols, 7), exp_noise(rows, cols, 7),
                      exp_noise(5 * rows, cols, 9)[4 * rows: 5 * rows], exp_noise(3 * rows, cols, 8)[rows: 2 * rows]])
    assert torch.equal(got, want)
    assert sorted(cache) == sorted({(3, rows, cols, 7), (1, rows, cols, 7), (5, rows, cols, 9), (3, rows, cols, 8)})


@pytest.mark.parametrize("nb", [(2, 2), (2, -1), (0, 0), (-1, 0)])
def test_a_noise_batch_without_its_row_is_refused(nb):
    with pytest.raises(ValueError, match="noise_batch"):
        _nreq(nb)


def test_noise_batch_limits():
    check_noise_batch(_nreq((4, 3)), 4, max_batch=4)
    with pytest.raises(ValueError, match="max_batch"):
        check_noise_batch(_nreq((5, 0)), 4, max_batch=4)
    # a code row keeps the penalty while all its num_vq rows are below max_input_ids (625: rows 0..624)
    check_noise_batch(_nreq((200, 155), penalty=625), 4)
    with pytest.raises(ValueError, match="penalty"):
        check_noise_batch(_nreq((200, 156), penalty=625), 4)
    check_noise_batch(_nreq((200, 156)), 4)  # no penalty: any row
    # a text request (one row) is checked when it is made
    _nreq((4, 2), text=True, penalty=3)
    with pytest.raises(ValueError, match="penalty"):
        _nreq((4, 3), text=True, penalty=3)
