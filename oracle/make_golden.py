"""Generate tests/golden/*.npz by running the REFERENCE ITSELF (build container only).

    python -m oracle.make_golden

Inputs are the seeded synthetic weights/prompts of chattts_b200.synth / .prompts (identical on
every box); outputs are what ``/root/reference``'s own ``GPT.generate`` / ``DVAE`` produce on
them with stubs for the three absent third-party packages (oracle/ref_import.py).  The GPU
parity tests load these files, so they do not need the reference at run time.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from chattts_b200.config import Config
from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_dvae_state, synth_embed_state, synth_gpt_state
from oracle.ref_models import build_reference_dvae, build_reference_gpt, reference_generate

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

GPT_CASES = {
    # name: (lengths, prompt_seed, sampler_seed, steps, kwargs)
    "gpt_audio_b1": ([16], 1, 1234, 24, {}),
    "gpt_audio_b3_ragged": ([5, 12, 9], 1, 42, 16, {}),
    "gpt_audio_b2_nopenalty_topk5": ([8, 8], 2, 7, 12, dict(repetition_penalty=1.0, top_K=5, top_P=0.9)),
    "gpt_text_b2": ([7, 4], 3, 7, 8, dict(text=True)),
}


def gen_gpt():
    gs, es = synth_gpt_state(0), synth_embed_state(1)
    gpt, embed = build_reference_gpt(gs, es)
    for name, (lengths, pseed, sseed, steps, kw) in GPT_CASES.items():
        ids, mask, tmask = synth_prompt_batch(lengths, seed=pseed)
        if kw.get("text"):
            ref = reference_generate(gpt, embed, ids, mask, tmask, temperature=[0.7], eos_token=21001,
                                     max_new_token=steps, repetition_penalty=1.0, num_code=21178, infer_text=True,
                                     return_hidden=False, manual_seed=sseed)
            hid = np.zeros((0,), np.float32)
        else:
            ref = reference_generate(gpt, embed, ids, mask, tmask, temperature=[0.3] * 4, eos_token=625,
                                     max_new_token=steps, min_new_token=steps, manual_seed=sseed,
                                     top_P=kw.get("top_P", 0.7), top_K=kw.get("top_K", 20),
                                     repetition_penalty=kw.get("repetition_penalty", 1.05))
            hid = torch.stack([h for h in ref.hiddens]).numpy()
        lens = np.array([len(i) for i in ref.ids])
        pad = np.full((len(lengths), steps, 4), -1, np.int64)
        for b, t in enumerate(ref.ids):
            pad[b, : len(t)] = t.numpy() if t.dim() == 2 else t.numpy()[:, None]
        np.savez_compressed(os.path.join(OUT, name + ".npz"), lengths=np.array(lengths), prompt_seed=pseed,
                            sampler_seed=sseed, steps=steps, ids=pad, n=lens, hiddens=hid.astype(np.float32))
        print(name, lens, pad[0, :2].tolist())


def gen_sampler():
    """Rows of logits pushed through the reference's own processor objects + torch.multinomial."""
    from oracle.ref_import import load_reference

    load_reference()
    from ChatTTS.model import gen_logits

    g = torch.Generator().manual_seed(11)
    rows, V, n_gen = 16, 626, 20
    logits = torch.randn(rows, V, generator=g) * 2.0
    gen_ids = torch.randint(0, 40, (rows, n_gen), generator=g)  # small id range => repeats in the window
    temp = torch.tensor([0.3, 0.5, 0.7, 1.0])
    out = {}
    for tag, (tp, tk, rp) in {"default": (0.7, 20, 1.05), "p95k3": (0.95, 3, 1.2), "nop": (None, 20, 1.0),
                              "nok": (0.5, None, 1.05)}.items():
        warp, proc = gen_logits(num_code=625, top_P=tp, top_K=tk, repetition_penalty=rp)
        x = logits / temp.repeat(rows // 4)[:, None]
        for pr in (*proc, *warp):
            x = pr(gen_ids, x)
        scores = torch.softmax(x, -1)
        idx = torch.multinomial(scores, 1, generator=torch.Generator().manual_seed(99))
        out["idx_" + tag] = idx[:, 0].numpy()
        out["keep_" + tag] = torch.isfinite(x).numpy()
    np.savez_compressed(os.path.join(OUT, "sampler_rows.npz"), logits=logits.numpy(), gen_ids=gen_ids.numpy(),
                        temperature=temp.numpy(), seed=99, **out)
    print("sampler", {k: v[:6].tolist() for k, v in out.items() if k.startswith("idx")})


def gen_dvae():
    cfg = Config()
    st = synth_dvae_state(2, cfg.decoder, cfg.decoder.idim)
    ref = build_reference_dvae(st, cfg.decoder, cfg.decoder.idim)
    g = torch.Generator().manual_seed(21)
    x = torch.randn(2, 768, 12, generator=g)
    with torch.no_grad():
        mel = ref(x.clone(), "decode")
    np.savez_compressed(os.path.join(OUT, "dvae_decoder_hidden.npz"), x=x.numpy(), mel=mel.numpy())
    print("dvae", mel.shape, float(mel.abs().mean()))


def gen_dvae_encode():
    """Encode branch: mel and encoder output from the REFERENCE's modules (torchaudio mel, downsample convs, encoder
    stack); ids / margins from the oracle's FSQ restatement applied to the reference's encoder output (third-party
    quantiser absent - parity unpinned for that last step)."""
    from chattts_b200.synth import synth_speech_like
    from oracle.dvae_oracle import fsq_quantize
    from oracle.ref_models import build_reference_dvae_encoder

    cfg = Config()
    st = synth_dvae_state(3, cfg.dvae.decoder, cfg.dvae.decoder.idim, cfg.dvae.vq, encoder=cfg.dvae.encoder)
    ref = build_reference_dvae_encoder(st, cfg.dvae.decoder, cfg.dvae.encoder, cfg.dvae.decoder.idim)
    seconds, seed = 1.37, 7                      # 32 880 samples: not a multiple of the hop, odd frame count
    wav = synth_speech_like(seconds, seed)
    with torch.inference_mode():
        mel = ref.preprocessor_mel(wav.clone())
        mel = mel / ref.coef.view(100, 1)
        x = ref.encoder(ref.downsample_conv(mel).unsqueeze(0))
    ids, margin = fsq_quantize(x.transpose(1, 2).clone(), st)
    np.savez_compressed(os.path.join(OUT, "dvae_encode.npz"), seconds=seconds, seed=seed, mel_over_coef=mel.numpy(),
                        ids=ids.numpy().astype(np.int32), margin=margin.numpy())
    print("dvae encode", tuple(ids.shape), "frames", mel.shape[1], "min margin", float(margin.min()))


ENCODE_CASES = ((1.3, 0), (2.0, 1))     # (seconds, seed) of synth_speech_like
ENCODE_CHANNELS = 96                     # encoder-output channels stored per case (a fixed, seeded sample of 1024)


def encode_channel_sample() -> torch.Tensor:
    return torch.randperm(1024, generator=torch.Generator().manual_seed(1024))[:ENCODE_CHANNELS].sort().values


def gen_reference_checks():
    """What tests/test_oracle_vs_reference.py compares the oracle against: the reference's GPT.generate (audio and text),
    Embed, DVAE decode branch and encode-side modules, on seeded inputs."""
    from chattts_b200.synth import synth_speech_like
    from oracle.ref_models import build_reference_dvae_encoder

    out = {}
    gs, es = synth_gpt_state(0), synth_embed_state(1)
    gpt, embed = build_reference_gpt(gs, es)
    for tag, lengths, seed in (("audio_b1", [16], 1234), ("audio_b3", [5, 12, 9], 42)):
        ids, mask, tmask = synth_prompt_batch(lengths, seed=1)
        ref = reference_generate(gpt, embed, ids, mask, tmask, temperature=[0.3] * 4, eos_token=625,
                                 max_new_token=12, min_new_token=12, manual_seed=seed)
        out[tag + "_ids"] = torch.stack(list(ref.ids)).numpy()
        out[tag + "_hiddens"] = torch.stack(list(ref.hiddens)).numpy()
    ids, mask, tmask = synth_prompt_batch([7, 4], seed=3)
    ref = reference_generate(gpt, embed, ids, mask, tmask, temperature=[0.7], eos_token=21001, max_new_token=6,
                             repetition_penalty=1.0, num_code=21178, infer_text=True, return_hidden=False, manual_seed=7)
    out["text_n"] = np.array([len(t) for t in ref.ids])
    out["text_ids"] = np.full((2, 6), -1, np.int64)
    for b, t in enumerate(ref.ids):
        out["text_ids"][b, : len(t)] = t.reshape(len(t), -1)[:, 0].numpy()
    ids, mask, tmask = synth_prompt_batch([6, 3], seed=5)
    tmask[0, -2:] = False  # mixed text / code positions (audio prompt splice, tokenizer.py:115-124)
    ids[0, -2:] = torch.randint(0, 626, (2, 4), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        out.update(embed_ids=ids.numpy(), embed_tmask=tmask.numpy(), embed_out=embed(ids, tmask).numpy())

    cfg = Config()
    st = synth_dvae_state(2, cfg.decoder, cfg.decoder.idim)
    x = torch.randn(2, 768, 20, generator=torch.Generator().manual_seed(20))
    with torch.no_grad():
        out.update(dvae_x=x.numpy(), dvae_mel=build_reference_dvae(st, cfg.decoder, cfg.decoder.idim)(x.clone(), "decode").numpy())

    st = synth_dvae_state(3, cfg.dvae.decoder, cfg.dvae.decoder.idim, cfg.dvae.vq, encoder=cfg.dvae.encoder)
    ref = build_reference_dvae_encoder(st, cfg.dvae.decoder, cfg.dvae.encoder, cfg.dvae.decoder.idim)
    chans = encode_channel_sample()
    for i, (seconds, seed) in enumerate(ENCODE_CASES):
        wav = synth_speech_like(seconds, seed)
        with torch.inference_mode():
            mel = ref.preprocessor_mel(wav.clone())
            x = ref.encoder(ref.downsample_conv(mel / ref.coef.view(100, 1)).unsqueeze(0))
        out[f"encode{i}_mel"] = mel.numpy()
        out[f"encode{i}_x_shape"] = np.array(x.shape)
        out[f"encode{i}_x"] = x[:, chans].numpy()
    np.savez_compressed(os.path.join(OUT, "reference_checks.npz"), **out)
    print("reference checks", {k: v.shape for k, v in out.items()})


def gen_host_checks():
    """What the host-logic tests compare against: the reference's Normalizer, Speaker and Tokenizer outputs, and its
    spk_stat asset (tests/golden/host_reference.json, tests/golden/speaker_apply.npz)."""
    import json
    import re
    import tempfile

    from oracle.ref_import import REFERENCE_ROOT, load_reference

    import sys

    sys.path.insert(0, os.path.dirname(OUT))  # the inputs are defined by the tests that use these outputs
    import test_norm_audio as tn
    import test_speaker as ts
    import test_tokenizer as tt

    load_reference()
    from ChatTTS.model.speaker import Speaker as RefSpeaker
    from ChatTTS.model.tokenizer import Tokenizer as RefTokenizer
    from ChatTTS.norm import Normalizer as RefNormalizer

    out = {}
    cfg_src = open(os.path.join(REFERENCE_ROOT, "ChatTTS", "config", "config.py"), encoding="utf-8").read()
    out["spk_stat"] = re.search(r'spk_stat: str = \(\s*"([^"]+)"', cfg_src).group(1)

    fd, path = tempfile.mkstemp(suffix=".json")
    with os.fdopen(fd, "w", encoding="utf-8") as f:
        json.dump(tn.HOMO, f, ensure_ascii=False)
    norm = RefNormalizer(path)
    os.unlink(path)
    assert norm.register("en", lambda s: s.upper())
    out["normalizer"] = [[text, nm, homo, lang, norm(text, nm, homo, lang)]
                         for text in tn.CASES for nm in (True, False) for homo in (True, False) for lang in (None, "zh", "en")]

    ref = object.__new__(RefSpeaker)
    emb, vec, ids = ts.apply_inputs()
    applied = ref.apply(emb.clone(), vec, ids, 21143, torch.device("cpu"))
    np.savez_compressed(os.path.join(OUT, "speaker_apply.npz"), applied=applied.numpy())
    deco = []
    for spk_emb, smp in ((None, None), ("x", None), ("x", "sample text")):
        t = ["  hi [Stts] there[spk_emb] ", "[empty_spk]b"]
        deco.append([spk_emb, smp, ref.decorate_code_prompts(t, "[speed_5]", smp, spk_emb), t])
    out["decorate_code"] = deco
    out["decorate_text"] = ref.decorate_text_prompts(["a", "b"], "[oral_2]")

    with tempfile.TemporaryDirectory() as d:
        import pathlib

        tok = RefTokenizer(tt._write_vocab(pathlib.Path(d)))
        if not hasattr(tok._tokenizer, "encode_plus"):       # API drift: transformers >= 5 removed encode_plus
            tok._tokenizer.encode_plus = tok._tokenizer.__call__
        out["tokenizer_attrs"] = [tok.len, tok.spk_emb_ids, tok.break_0_ids, tok.eos_token]
        enc = []
        for prompt in (None, tt.PROMPT):
            enc.append([[str(x.dtype), x.tolist()] for x in tok.encode(list(tt.TEXTS), 4, prompt=None if prompt is None else prompt.clone())])
        out["tokenizer_encode"] = enc
        out["tokenizer_decode"] = tok.decode(tt.DECODE_SEQ)
    with open(os.path.join(OUT, "host_reference.json"), "w", encoding="utf-8") as f:
        json.dump(out, f, ensure_ascii=False, indent=0)
    print("host checks", len(out["normalizer"]), "normalizer cases")


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    gen_gpt()
    gen_sampler()
    gen_dvae()
    gen_dvae_encode()
    gen_reference_checks()
    gen_host_checks()
