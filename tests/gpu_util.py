import gc
import os

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.config import Config
from chattts_b200.embed import Embed
from chattts_b200.gpt import GPT
from chattts_b200.synth import synth_embed_state, synth_gpt_state

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_cache = {}


def build_gpt(seed=0, std=0.02, max_batch=32, max_context=640):
    key = (seed, std, max_batch, max_context)
    if key not in _cache:
        cfg = Config()
        gs, es = synth_gpt_state(seed, std), synth_embed_state(seed + 1)
        embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                      cfg.embed.num_vq).load_state_dict(es).to("cuda")
        gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=max_batch, max_context=max_context)
        gpt.load_state(gs)
        _cache[key] = (gpt, embed, gs, es)
    return _cache[key]


def load_gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def release_on_teardown(*caches):
    """A module-scoped autouse fixture that empties ``caches`` (the module's dicts of engine handles, models and device
    tensors) once its tests are done, so that the device memory they hold is free for the modules that run after it.
    Assign it to a module-level name: ``_release = release_on_teardown(_models, _refs)``."""

    @pytest.fixture(scope="module", autouse=True)
    def _release():
        yield
        for c in caches:
            c.clear()
        gc.collect()
        if torch.cuda.is_available():
            torch.cuda.synchronize()
            torch.cuda.empty_cache()

    return _release


# the environment variables that take a decode step away from a handle created with them
_STEP_OFF = {_lib.STEP_FLOW_INK: ("CTB_NO_FLOW", "CTB_FLOW_NO_INK"), _lib.STEP_FLOW: ("CTB_NO_FLOW",),
             _lib.STEP_MEGA: ("CTB_NO_MEGA",), _lib.STEP_WGMMA: ("CTB_GPT_FMA",), _lib.STEP_FMA: ()}


def expect_step(gpt, B, want, infer_text=False):
    """Assert that the decode step ``want`` (a _lib.STEP_* value) serves a static batch of ``B`` rows on ``gpt``'s
    handle.  Skips, with the reason, when the device or the environment the tests started with rules that step out:
    k_flow needs 128 .. 191 SMs and k_step at least 128 (ctb_gpt_create).  Call it with the environment as the tests
    started, not as a test set it for a handle."""
    got = _lib.step_kind(gpt._handle, B, infer_text)
    if got != want:
        sms = torch.cuda.get_device_properties(gpt.device_gpt).multi_processor_count
        if want in (_lib.STEP_FLOW_INK, _lib.STEP_FLOW) and not 128 <= sms <= 191:
            pytest.skip(f"k_flow needs 128..191 SMs; this device has {sms}")
        if want == _lib.STEP_MEGA and sms < 128:
            pytest.skip(f"k_step needs at least 128 SMs; this device has {sms}")
        off = [k for k in _STEP_OFF[want] if k in os.environ]
        if off:
            pytest.skip(f"{', '.join(off)} set in the environment: no {_lib.STEP_NAMES[want]} step")
    assert got == want, (B, infer_text, _lib.STEP_NAMES.get(got, got), _lib.STEP_NAMES[want])
