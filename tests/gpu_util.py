import gc
import os

import numpy as np
import pytest
import torch

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
