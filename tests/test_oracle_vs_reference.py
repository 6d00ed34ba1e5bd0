"""Pin oracle/gpt_oracle.py and oracle/dvae_oracle.py against the reference's own code, through what the reference computed
on seeded inputs (tests/golden/reference_checks.npz, written by oracle/make_golden.py gen_reference_checks)."""
import os

import numpy as np
import pytest
import torch

from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from oracle.gpt_oracle import GPTOracle, SamplerParams

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_checks.npz"))


@pytest.fixture(scope="module")
def orc():
    return GPTOracle(synth_gpt_state(0), synth_embed_state(1))


@pytest.mark.parametrize("lengths,seed", [([16], 1234), ([5, 12, 9], 42)])
def test_audio_generate_ids_and_hiddens(orc, lengths, seed):
    tag = f"audio_b{len(lengths)}"
    ids, mask, tmask = synth_prompt_batch(lengths, seed=1)
    out = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                       max_new_token=12, min_new_token=12, sampler=SamplerParams(), return_hidden=True,
                       manual_seed=seed)
    for b in range(len(lengths)):
        ref_ids, ref_h = GOLD[tag + "_ids"][b], GOLD[tag + "_hiddens"][b]
        assert np.array_equal(ref_ids, out.ids[b].numpy()), (b, ref_ids, out.ids[b])
        assert np.abs(ref_h - out.hiddens[b].numpy()).max() < 2e-5


def test_text_generate_ids(orc):
    ids, mask, tmask = synth_prompt_batch([7, 4], seed=3)
    out = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.7]), 21001, attention_mask=mask,
                       max_new_token=6, sampler=SamplerParams(repetition_penalty=1.0, penalty_max_ids=21178),
                       infer_text=True, manual_seed=7)
    for b in range(2):
        n = int(GOLD["text_n"][b])
        assert np.array_equal(out.ids[b].reshape(-1).numpy(), GOLD["text_ids"][b, :n])


def test_embed_prompt_matches(orc):
    ids, tmask = torch.from_numpy(GOLD["embed_ids"]), torch.from_numpy(GOLD["embed_tmask"])
    assert not bool(tmask[0, -2:].any()) and bool(tmask[0, :-2].all())  # mixed text / code positions
    assert np.array_equal(orc.embed_prompt(ids, tmask).numpy(), GOLD["embed_out"])


def test_dvae_decoder_branch_matches_reference():
    """DVAE(decoder_config, dim=384) decode branch (the default use_decoder=True path)."""
    from chattts_b200.config import Config
    from chattts_b200.synth import synth_dvae_state
    from oracle.dvae_oracle import dvae_decode

    cfg = Config()
    st = synth_dvae_state(2, cfg.decoder, cfg.decoder.idim)
    want = torch.from_numpy(GOLD["dvae_mel"])
    got = dvae_decode(torch.from_numpy(GOLD["dvae_x"]), st)
    assert want.shape == got.shape == (2, 100, 40)
    assert (want - got).abs().max() < 1e-5 * max(1.0, float(want.abs().max()))


def test_dvae_encode_branch_matches_reference_up_to_the_quantizer():
    """Encode branch (dvae.py:265-274) piece by piece against the reference's own modules: MelSpectrogramFeatures
    (torchaudio), downsample_conv, encoder stack (a fixed sample of its output channels is stored).  The FSQ quantiser
    itself is third-party and absent (parity unpinned)."""
    from chattts_b200.config import Config
    from chattts_b200.synth import synth_dvae_state, synth_speech_like
    from oracle.dvae_oracle import dvae_encode, mel_features
    from oracle.make_golden import ENCODE_CASES, encode_channel_sample

    cfg = Config()
    st = synth_dvae_state(3, cfg.dvae.decoder, cfg.dvae.decoder.idim, cfg.dvae.vq, encoder=cfg.dvae.encoder)
    chans = encode_channel_sample()
    for i, (seconds, seed) in enumerate(ENCODE_CASES):
        wav = synth_speech_like(seconds, seed)
        mel_ref, x_ref = torch.from_numpy(GOLD[f"encode{i}_mel"]), torch.from_numpy(GOLD[f"encode{i}_x"])
        mel = mel_features(wav)
        assert mel.shape == mel_ref.shape == (100, wav.numel() // 256 + 1)
        assert (mel - mel_ref).abs().max() < 2e-4          # same stft; the filterbank matmul runs in another order
        ids, margin, _, x = dvae_encode(wav, st, return_parts=True)
        assert tuple(x.shape) == tuple(GOLD[f"encode{i}_x_shape"]) == (1, 1024, (wav.numel() // 256 + 1) // 2)
        assert (x[:, chans] - x_ref).abs().max() < 1e-4 * max(1.0, float(x_ref.abs().max()))
        assert ids.shape == (1, 4, x.shape[2]) and int(ids.min()) >= 0 and int(ids.max()) < 625
