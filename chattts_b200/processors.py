"""Sampling-filter descriptors (reference ChatTTS/model/processors.py).

The reference builds callable HF warpers and applies them on the host
(processors.py:38-58, gpt.py:489-490).  Here the filters run inside the fused sampler
kernel, so these objects only *describe* the filter; they expose the same attribute names
as the reference / HF objects (``penalty``/``max_input_ids``/``past_window``,
``top_p``/``min_tokens_to_keep``, ``top_k``) so that either kind can be passed to
``GPT.generate(logits_processors=...)``.  Unknown callables raise: there is no host-side
fallback path.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

from ._lib import SamplerConfig


@dataclass
class CustomRepetitionPenaltyLogitsProcessorRepeat:
    """processors.py:7-35 (windowed ``penalty ** count``)."""

    penalty: float
    max_input_ids: int
    past_window: int

    def __post_init__(self):
        if not isinstance(self.penalty, float) or not (self.penalty > 0):
            raise ValueError(f"`penalty` has to be a strictly positive float, but is {self.penalty}")


@dataclass
class TopPLogitsWarper:
    top_p: float
    min_tokens_to_keep: int = 1

    def __post_init__(self):
        self.top_p = float(self.top_p)
        if self.top_p < 0 or self.top_p > 1.0:
            raise ValueError(f"`top_p` has to be a float > 0 and < 1, but is {self.top_p}")


@dataclass
class TopKLogitsWarper:
    top_k: int
    min_tokens_to_keep: int = 1

    def __post_init__(self):
        if not isinstance(self.top_k, int) or self.top_k <= 0:
            raise ValueError(f"`top_k` has to be a strictly positive integer, but is {self.top_k}")
        self.top_k = max(self.top_k, self.min_tokens_to_keep)


@dataclass
class ArgmaxOnly:
    """Extra processor for the 'greedy' benchmark config (SURVEY.md §8d C2): keep the row max.
    ``exclude_eos``: remove the EOS column first, so a forced-length run never ends up with an
    empty row when the arg-max is EOS and ``min_new_token`` bans it afterwards."""

    greedy: bool = True
    exclude_eos: bool = False


def gen_logits(num_code: int, top_P=0.7, top_K=20, repetition_penalty=1.0) -> Tuple[list, list]:
    """Same contract as processors.py:38-58: (warpers, processors)."""
    warpers: List[object] = []
    if top_P is not None:
        warpers.append(TopPLogitsWarper(top_P, min_tokens_to_keep=3))
    if top_K is not None:
        warpers.append(TopKLogitsWarper(top_K, min_tokens_to_keep=3))
    processors: List[object] = []
    if repetition_penalty is not None and repetition_penalty != 1:
        processors.append(CustomRepetitionPenaltyLogitsProcessorRepeat(repetition_penalty, num_code, 16))
    return warpers, processors


def build_sampler_config(logits_processors: Sequence[object], temperature: Sequence[float], eos_token: int,
                         min_new_token: int, philox_seed: int = 0) -> SamplerConfig:
    """Translate the processor tuple of ``GPT.generate`` into the kernel's config.

    Enforces the only order the fused kernel implements (the reference's, core.py:649):
    penalty -> top-p -> top-k [-> argmax-only]."""
    cfg = SamplerConfig()
    if len(temperature) > 8:
        raise ValueError("at most 8 codebooks")
    for i in range(8):
        cfg.temperature[i] = float(temperature[i % len(temperature)])
    cfg.top_p, cfg.top_k, cfg.min_tokens_to_keep = -1.0, 0, 1
    cfg.penalty_on, cfg.past_window, cfg.penalty_max_ids, cfg.greedy = 0, 0, 0, 0
    stage = 0
    for proc in logits_processors:
        if hasattr(proc, "penalty") and hasattr(proc, "past_window") and hasattr(proc, "max_input_ids"):
            kind = 1
            if proc.past_window > 31:
                raise ValueError("past_window > 31 not supported")
            cfg.penalty_on = 1
            cfg.past_window = int(proc.past_window)
            cfg.penalty_max_ids = int(proc.max_input_ids)
            # same call as processors.py:28 -> identical fp32 alpha values
            lut = torch.pow(proc.penalty, torch.arange(32))
            for i in range(32):
                cfg.penalty_lut[i] = float(lut[i])
        elif hasattr(proc, "top_p"):
            kind = 2
            cfg.top_p = float(proc.top_p)
            cfg.min_tokens_to_keep = int(getattr(proc, "min_tokens_to_keep", 1))
            # HF: `cumulative_probs <= (1 - self.top_p)` - the python double 1 - top_p, cast to the fp32 of the tensor
            cfg.top_p_removed_max = 1.0 - float(proc.top_p)
            cfg.has_removed_max = 1
        elif hasattr(proc, "top_k"):
            kind = 3
            cfg.top_k = int(proc.top_k)  # HF already folded max(top_k, min_tokens_to_keep)
        elif getattr(proc, "greedy", False):
            kind = 4
            cfg.greedy = 2 if getattr(proc, "exclude_eos", False) else 1
        else:
            raise TypeError(
                f"unsupported logits processor {type(proc).__name__}: the GPU sampler implements the reference's "
                "repetition-penalty / top-p / top-k filters only (no host fallback)")
        if kind <= stage:
            raise ValueError("logits processors must be ordered penalty -> top-p -> top-k (reference core.py:649)")
        stage = kind
    cfg.eos_token = int(eos_token)
    cfg.min_new_token = int(min_new_token)
    cfg.philox_seed = int(philox_seed) & 0xFFFFFFFFFFFFFFFF
    return cfg


def exp_noise(rows: int, cols: int, seed: int) -> torch.Tensor:
    """Exp(1) noise of ``torch.multinomial`` under ``generator.manual_seed(seed)``
    (gpt.py:504-508: re-seeded every step => one constant tensor per generate call)."""
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    return torch.empty(rows, cols, dtype=torch.float32).exponential_(1, generator=g)
