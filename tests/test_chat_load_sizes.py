"""``Chat.load`` passes the handle sizes (``max_batch``, ``max_context``) through to ``load_states``, with
``load_states``' defaults when they are not given (CPU: ``load_states`` is replaced by a recorder)."""
import numpy as np
import pytest
import torch

from test_load_glue import _make_assets


@pytest.mark.parametrize("kw,want", [({}, (32, 4096)), ({"max_batch": 64, "max_context": 640}, (64, 640))])
def test_chat_load_passes_handle_sizes_to_load_states(tmp_path, monkeypatch, kw, want):
    from chattts_b200 import Chat, b14

    c = Chat()
    _make_assets(tmp_path)
    seen = {}

    def fake_load_states(states, tokenizer, speaker, device=None, coef=None, **rest):
        seen.update(rest)
        return True

    monkeypatch.setattr(c, "load_states", fake_load_states)
    stat = b14.encode_to_string(np.concatenate([np.ones(768, np.float16), np.zeros(768, np.float16)]).tobytes())
    assert c.load(source="custom", custom_path=str(tmp_path), device=torch.device("cpu"), spk_stat=stat, **kw) is True
    assert (seen["max_batch"], seen["max_context"]) == want
