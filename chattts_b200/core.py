"""``Chat`` - the public API of the reference (ChatTTS/core.py) re-hosted on the H100 hot paths.

Same surface: ``Chat.load / infer / interrupt / unload / has_loaded / sample_random_speaker``,
``Chat.RefineTextParams`` / ``Chat.InferCodeParams`` (core.py:137-273).  The two hot paths are
ours (``GPT.generate`` -> chattts_b200.gpt, ``_decode_to_wavs`` -> chattts_b200.decoder); the
out-of-scope host components (text normaliser, BERT tokenizer, speaker strings, asset download -
SURVEY.md 2 rows 7, 8, 10, 11) are *injected*: ``load()`` takes them from an installed reference
``ChatTTS`` package, ``load_states()`` accepts any objects with the same methods (tests use stubs).
"""
from __future__ import annotations

import copy
import logging
import os
import queue
import re
from dataclasses import dataclass, replace
from typing import Dict, List, Optional, Union

import numpy as np
import torch

from . import _lib
from .config import Config
from .decoder import ENC_NFFT, decode_to_wavs_window, DVAE, Vocos, decode_to_wavs, stream_window
from .embed import Embed
from .engine import Job, OpenEngine, SlotImage, check_prefill_budget
from .gpt import GPT
from .norm import Normalizer
from .processors import gen_logits


def split_sentences(text: str) -> List[str]:
    """``infer``'s sentence split (``split_text=True``): the lines of a text with a newline, else its sentences
    ending in '。' or '. ' (reference core.py:237-241)."""
    if "\n" in text:
        return text.split("\n")
    return [t for t in re.split(r"(?<=。)|(?<=\.\s)", text) if t]


class Chat:
    def __init__(self, logger=logging.getLogger(__name__)):
        self.logger = logger
        self.config = Config()
        self.normalizer = Normalizer(logger=logger)        # no homophone map until load() finds the asset (core.py:39-42)
        self.context = GPT.Context()

    # core.py:49-64
    def has_loaded(self, use_decoder=False):
        check = ["vocos", "gpt", "tokenizer", "embed", "decoder" if use_decoder else "dvae"]
        for module in check:
            if not hasattr(self, module):
                self.logger.warning(f"{module} not initialized.")
                return False
        return True

    # ------------------------------------------------------------------ loading
    def load(self, source="local", force_redownload=False, compile: bool = False, custom_path=None,
             device: Optional[torch.device] = None, coef: Optional[torch.Tensor] = None, use_flash_attn=False,
             use_vllm=False, experimental: bool = False, spk_stat: Optional[str] = None, max_batch: int = 32,
             max_context: int = 4096) -> bool:
        """core.py:137-163.  ``compile`` / ``use_flash_attn`` / ``use_vllm`` / ``experimental`` are accepted and
        ignored (one back end, SURVEY.md quirk Q14).  The asset files are located like the reference does for
        ``source="local"`` (working directory or ``custom_path``) and ``"custom"``; downloading / sha256 checking
        (core.py:66-135) is left to the reference package, which ``source="huggingface"`` therefore still needs.
        ``spk_stat`` (config.py:132, the base16384 std|mean table random speakers are drawn from) is taken from the
        argument, else from an importable reference package; without it only ``sample_random_speaker`` is unavailable.
        ``max_batch`` / ``max_context`` size the handles as in ``load_states``: a slot engine serves up to
        ``max_batch`` slots (up to 64 on the wgmma step, half-precision engines included)."""
        root = self.download_models(source, force_redownload, custom_path)
        if root is None:
            return False
        from dataclasses import asdict

        paths = {k: os.path.join(root, v) for k, v in asdict(self.config.path).items()}
        from safetensors.torch import load_file
        from transformers import LlamaModel

        from .speaker import Speaker
        from .tokenizer import Tokenizer

        gpt_model = LlamaModel.from_pretrained(paths["gpt_ckpt_path"])
        states = {
            "gpt": {k: v for k, v in gpt_model.state_dict().items() if not k.startswith("embed_tokens")},
            "embed": load_file(paths["embed_path"]), "decoder": load_file(paths["decoder_ckpt_path"]),
            "dvae": load_file(paths["dvae_ckpt_path"]), "vocos": load_file(paths["vocos_ckpt_path"]),
        }
        homophones = None
        if spk_stat is None or homophones is None:
            try:
                import ChatTTS as ref  # optional: only its data constants are read

                spk_stat = spk_stat or ref.config.Config().spk_stat
                cand = os.path.join(os.path.dirname(ref.__file__), "res", "homophones_map.json")   # core.py:39-42
                homophones = cand if os.path.exists(cand) else None
            except Exception:
                pass
        dev = device or torch.device("cuda")
        self.normalizer = Normalizer(homophones, self.logger)
        return self.load_states(states, tokenizer=Tokenizer(paths["tokenizer_path"]),
                                speaker=Speaker(self.config.gpt.hidden_size, spk_stat, dev), device=dev, coef=coef,
                                max_batch=max_batch, max_context=max_context)

    def download_models(self, source="local", force_redownload=False, custom_path=None) -> Optional[str]:
        """core.py:66-135, without the downloader: returns the folder that holds ``asset/`` or ``None``."""
        if source == "huggingface":
            try:
                import ChatTTS as ref
            except Exception as e:  # pragma: no cover - needs the reference + network
                raise RuntimeError('source="huggingface" downloads through the reference package, which is not '
                                   'installed; fetch the assets yourself and use source="custom"') from e
            return ref.Chat(self.logger).download_models(source, force_redownload, custom_path)
        root = custom_path if custom_path is not None else os.getcwd()
        from dataclasses import asdict

        missing = [v for v in asdict(self.config.path).values() if not os.path.exists(os.path.join(root, v))]
        if missing:
            self.logger.error("assets missing under %s: %s", root, ", ".join(missing))
            return None
        return str(root)

    def load_states(self, states: Dict[str, Dict[str, torch.Tensor]], tokenizer, speaker, device=None, coef=None,
                    max_batch: int = 32, max_context: int = 4096, weights_blob: Optional[torch.Tensor] = None) -> bool:
        """Build every model from in-memory state dicts (reference names, SURVEY.md 8b) - core.py:275-384."""
        device = torch.device(device or "cuda")
        self.device = self.device_gpt = device
        cfg = self.config
        self.vocos = Vocos(cfg.vocos, device, max_batch=max_batch, max_tokens=max_context)
        self.vocos.state = {k: v.float() for k, v in states["vocos"].items()}
        self.dvae = DVAE(cfg.dvae.decoder, cfg.dvae.encoder, cfg.dvae.vq, dim=cfg.dvae.decoder.idim, coef=coef,
                         device=device, vocos=self.vocos, max_batch=max_batch, max_tokens=max_context)
        self.dvae.load_state_dict(states["dvae"])
        self.embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                           cfg.embed.num_vq).load_state_dict(states["embed"]).to(device)
        self.gpt = GPT(cfg.gpt, self.embed, device=device, device_gpt=device, logger=self.logger,
                       max_batch=max_batch, max_context=max_context)
        self.gpt.load_state(states.get("gpt"), weights_blob=weights_blob)
        self.speaker = speaker
        self.decoder = DVAE(cfg.decoder, dim=cfg.decoder.idim, coef=coef, device=device, vocos=self.vocos,
                            max_batch=max_batch, max_tokens=max_context)
        self.decoder.load_state_dict(states["decoder"])
        self.tokenizer = tokenizer
        self.coef = coef
        return self.has_loaded()

    def unload(self):
        logger = self.logger
        for module in ["vocos", "gpt", "decoder", "dvae", "tokenizer", "embed", "speaker"]:
            if hasattr(self, module):
                delattr(self, module)
        self.__init__(logger)

    def sample_random_speaker(self) -> str:
        return self.speaker.sample_random()

    def sample_audio_speaker(self, wav) -> str:
        """core.py:179-180: wav (24 kHz, 1-D) -> DVAE codes -> speaker-prompt string for ``InferCodeParams.spk_smp``."""
        if self.dvae.audio_encoder is None:
            raise RuntimeError("this DVAE checkpoint carries no encoder / VQ weights: cannot sample a speaker from audio")
        return self.speaker.encode_prompt(self.dvae.sample_audio(wav))

    # ------------------------------------------------------------------ params (core.py:182-206)
    @dataclass(repr=False, eq=False)
    class RefineTextParams:
        prompt: str = ""
        top_P: float = 0.7
        top_K: int = 20
        temperature: float = 0.7
        repetition_penalty: float = 1.0
        max_new_token: int = 384
        min_new_token: int = 0
        show_tqdm: bool = True
        ensure_non_empty: bool = True
        manual_seed: Optional[int] = None

    @dataclass(repr=False, eq=False)
    class InferCodeParams(RefineTextParams):
        prompt: str = "[speed_5]"
        spk_emb: Optional[str] = None
        spk_smp: Optional[str] = None
        txt_smp: Optional[str] = None
        temperature: float = 0.3
        repetition_penalty: float = 1.05
        max_new_token: int = 2048
        stream_batch: int = 24
        stream_speed: int = 12000
        pass_first_n_batches: int = 2

    # ------------------------------------------------------------------ infer (core.py:208-270)
    def infer(self, text, stream=False, lang=None, skip_refine_text=False, refine_text_only=False, use_decoder=True,
              do_text_normalization=True, do_homophone_replacement=True, split_text=True, max_split_batch=4,
              params_refine_text=None, params_infer_code=None):
        params_refine_text = params_refine_text or Chat.RefineTextParams()
        params_infer_code = params_infer_code or Chat.InferCodeParams()
        self.context.set(False)
        if split_text and isinstance(text, str):
            text = split_sentences(text)
            self.logger.info("split text into %d parts", len(text))
        if len(text) == 0:
            return []
        res_gen = self._infer(text, stream, lang, skip_refine_text, refine_text_only, use_decoder,
                              do_text_normalization, do_homophone_replacement, split_text, max_split_batch,
                              params_refine_text, params_infer_code)
        if stream:
            return res_gen
        if not refine_text_only:
            stripped = []
            thr = np.float32(1e-5)
            for wavs in res_gen:
                for wav in wavs:
                    stripped.append(wav[np.abs(wav) > thr])  # quirk Q20
            if split_text:
                return [np.concatenate(stripped)]
            return stripped
        return next(res_gen)

    def infer_continuous(self, texts, params_infer_code=None, use_decoder=True, slots=None, stream=False, lang=None,
                         skip_refine_text=True, do_text_normalization=True, do_homophone_replacement=True,
                         params_refine_text=None, refine_on_engine=False, split_text=False, max_split_batch=1,
                         dtype=torch.float32, prefill_budget: Optional[int] = None,
                         kv_pool_bytes: Optional[int] = None):
        """Synthesise many texts with continuous batching: each text is one job on an open slot engine
        (``open_engine``), all queued at once; ``params_infer_code`` is one ``InferCodeParams`` for all texts or a list
        with one per text (speaker, seed, temperature, top-P/K, penalty, token limits).  Generator of ``(index, wav)``
        in completion order; ``wav`` is what ``infer([texts[index]], split_text=False, skip_refine_text=True)``
        returns for that text with its params.  A code prompt (text plus ``spk_smp``) may be up to ``max_context`` -
        ``max_new_token`` tokens; over 1,024 tokens it is prefilled with the tiled attention kernel, whose ids equal
        ``infer``'s except at the sampler's near-ties (``GPT.generate_continuous``).
        Normalisation and the optional text refinement run as in ``infer``; ``params_refine_text`` is one
        ``RefineTextParams`` or one per text.

        With ``skip_refine_text=False`` the texts are refined first, in static batches of up to ``max_batch`` texts,
        and no speech code starts before every text is refined.  ``refine_on_engine=True`` refines each text as a
        request of its own on the slot engine instead, and its speech codes follow as soon as its refinement ends:
        ``wav`` is then what ``infer([texts[index]], split_text=False, skip_refine_text=False)`` returns with that
        text's params.  A seeded refinement depends on the batch it is drawn in, so the two modes give different
        seeded results; the batched one stays the default.

        ``split_text=True`` makes each text a paragraph, split into sentences as ``infer`` splits it, with one voice
        across its sentences (see ``ChatEngine.submit``): ``wav`` is then what ``infer(texts[index], split_text=True,
        max_split_batch=max_split_batch, skip_refine_text=True)[0]`` returns with that text's params, which are not
        modified; with ``skip_refine_text=False`` each sentence is refined on the engine first, and ``wav`` is what
        ``infer(texts[index], max_split_batch=max_split_batch, params_refine_text=...)[0]`` returns (seeded: bit for
        bit on the code path).

        ``slots`` defaults to max(2, min(max_batch, len(texts))), with ``split_text`` to the handle's ``max_batch``
        (``load(max_batch=...)``); engines of 9..64 slots run the wgmma decode step.  ``Chat.interrupt()`` ends the running texts with what they have, or with ``split_text`` cancels every
        unfinished paragraph (see ``_continuous``).

        ``dtype=torch.float16`` runs every request on a half-precision engine (``GPT.generate_continuous``): fp16
        layer weights and KV cache, as the reference's ``use_vllm=True`` serves; the waveforms then follow that model.
        It serves up to 64 slots.  Path 2 (DVAE / Vocos) is unchanged.

        ``prefill_budget`` (prompt columns per poll, at least 128; default None) bounds the prefill the running texts
        wait for at each poll: a prompt that does not fit, such as one with a long ``spk_smp``, is prefilled in chunks
        over several polls with the same results (``GPT.generate_continuous``).

        ``kv_pool_bytes`` (default None) bounds the engine's KV memory: slots take pages from a pool of that many bytes
        as they grow, and a running request the pool cannot cover is suspended to host memory and resumed later with
        the same results (``GPT.generate_continuous``)."""
        _lib.engine_flags(dtype)  # an unsupported dtype raises here, before any device work
        check_prefill_budget(prefill_budget)
        if stream:
            raise ValueError("infer_continuous: stream=True is not supported; each waveform is yielded when complete "
                             "(infer_continuous_stream streams)")
        texts, params = self._continuous_params(texts, params_infer_code)
        return self._continuous(texts, params, self._refine_params(texts, params_refine_text), False, use_decoder,
                                slots, lang, skip_refine_text, do_text_normalization, do_homophone_replacement,
                                refine_on_engine, split_text, max_split_batch, dtype, prefill_budget, kv_pool_bytes)

    def infer_continuous_stream(self, texts, params_infer_code=None, use_decoder=True, slots=None, lang=None,
                                skip_refine_text=True, do_text_normalization=True, do_homophone_replacement=True,
                                params_refine_text=None, refine_on_engine=False, split_text=False, max_split_batch=1,
                                dtype=torch.float32, prefill_budget: Optional[int] = None,
                                kv_pool_bytes: Optional[int] = None):
        """Streaming synthesis of many texts with continuous batching on an open slot engine.  Generator of ``(index,
        chunk, last)``, ``chunk`` a ``[1, n]`` float32 array; for each text the chunks are those ``infer([texts[index]], stream=True, split_text=False, skip_refine_text=True)`` yields with that
        text's params (its own ``stream_batch``, ``stream_speed`` and ``pass_first_n_batches``), and ``last`` marks
        its final chunk.  A seeded text whose first code is EOS yields one empty final chunk.  All windows due at one
        engine poll are decoded in one ragged call (``TokenDecoder.decode_rows``), straight from the engine's
        buffers.  Arguments as for ``infer_continuous``; with ``refine_on_engine=True`` the chunks are those of
        ``infer([texts[index]], stream=True, split_text=False, skip_refine_text=False)``.  With ``split_text=True``
        each text is a paragraph, streamed sentence by sentence as ``ChatEngine.submit(split_text=True,
        stream=True)`` streams it, refined first with ``skip_refine_text=False``.  ``dtype``, ``prefill_budget`` and
        ``kv_pool_bytes`` as in ``infer_continuous``; neither of the last two changes the chunks."""
        _lib.engine_flags(dtype)
        check_prefill_budget(prefill_budget)
        texts, params = self._continuous_params(texts, params_infer_code)
        return self._continuous(texts, params, self._refine_params(texts, params_refine_text), True, use_decoder,
                                slots, lang, skip_refine_text, do_text_normalization, do_homophone_replacement,
                                refine_on_engine, split_text, max_split_batch, dtype, prefill_budget, kv_pool_bytes)

    def refine_continuous(self, texts, params_refine_text=None, slots=None, lang=None, do_text_normalization=True,
                          do_homophone_replacement=True, dtype=torch.float32, kv_pool_bytes: Optional[int] = None):
        """Refine many texts on the slot engine, each as a request of its own: generator of ``(index, refined_text)``
        in completion order.  ``refined_text`` is what ``infer([texts[index]], refine_text_only=True,
        split_text=False, params_refine_text=...)[0]`` returns for that text; ``params_refine_text`` is one
        ``RefineTextParams`` or one per text.  ``dtype`` and ``kv_pool_bytes`` as in ``infer_continuous``."""
        _lib.engine_flags(dtype)
        if isinstance(texts, str):
            texts = [texts]
        texts = list(texts)
        refine = self._refine_params(texts, params_refine_text)
        assert self.has_loaded()
        self.context.set(False)
        if not texts:
            return
        texts = [self.normalizer(t, do_text_normalization, do_homophone_replacement, lang) for t in texts]
        requests = [self._refine_request(t, r) for t, r in zip(texts, refine)]
        for i, out in self.gpt.generate_continuous(requests, slots=slots, return_hidden=False, context=self.context,
                                                   dtype=dtype, kv_pool_bytes=kv_pool_bytes):
            yield i, self._refined_text(out)

    @staticmethod
    def _continuous_params(texts, params_infer_code):
        if isinstance(texts, str):
            texts = [texts]
        texts = list(texts)
        if isinstance(params_infer_code, (list, tuple)):
            if len(params_infer_code) != len(texts):
                raise ValueError("params_infer_code: one InferCodeParams per text")
            return texts, list(params_infer_code)
        return texts, [params_infer_code or Chat.InferCodeParams()] * len(texts)

    @staticmethod
    def _refine_params(texts, params_refine_text):
        if isinstance(params_refine_text, (list, tuple)):
            if len(params_refine_text) != len(texts):
                raise ValueError("params_refine_text: one RefineTextParams per text")
            return list(params_refine_text)
        return [params_refine_text or Chat.RefineTextParams()] * len(texts)

    def _continuous(self, texts, params, refine, stream, use_decoder, slots, lang, skip_refine_text,
                    do_text_normalization, do_homophone_replacement, refine_on_engine, split_text, max_split_batch,
                    dtype, prefill_budget=None, kv_pool_bytes=None):
        """``infer_continuous*``: every text one ``ChatEngine`` job on one open engine.  Generator of ``(index, wav)``
        in completion order, or of ``(index, chunk, last)`` as the chunks come.

        Batched refinement (``skip_refine_text=False`` without ``refine_on_engine`` or ``split_text``) refines the
        normalised texts in static batches of up to ``max_batch`` before the engine opens, and the refined texts are
        spoken as they are: they are not normalised again.  The first stage of every text is queued in one step, so
        the engine's first admission fills min(slots, len(texts)) slots.  ``slots`` defaults to max(2, min(max_batch,
        len(texts))), with ``split_text`` to ``max_batch``; the poll interval is CTB_DECODE_CHUNK, else 24 with
        ``split_text``, else the smallest ``stream_batch`` of the texts when streaming, else 32.

        ``Chat.interrupt()``: a text's audio ends early only where it has no later part to wait for.  Without
        ``split_text`` the engine stops at its first poll that sees the interrupt: every text whose speech stage is
        running ends with the tokens it has (its silence-stripped waveform, or its final chunk with ``last=True``),
        and a text still waiting or refining yields nothing.  With ``split_text`` a paragraph cut short would miss
        sentences, so within one poll every unfinished paragraph is cancelled and yields nothing more.  Either way
        "generation is interrupted" is logged and the generator ends with the handle free.  An invalid text raises
        here; closing the generator early or an error in the engine cancels every job and frees the handle too."""
        assert self.has_loaded(use_decoder=use_decoder)
        self.context.set(False)
        if not texts:
            return

        def normalize(t):
            return self.normalizer(t, do_text_normalization, do_homophone_replacement, lang)

        cap = max(p.max_new_token for p in params)
        if not skip_refine_text and (refine_on_engine or split_text):
            cap = max(cap, max(r.max_new_token for r in refine))
        elif not skip_refine_text:
            if any(r is not refine[0] for r in refine):
                raise ValueError("one RefineTextParams per text needs refine_on_engine=True (batched refinement "
                                 "draws every text of a batch with one set of parameters)")
            texts = [normalize(t) for t in texts]
            tokens = []
            for lo in range(0, len(texts), self.gpt.max_batch):
                refined = self._refine_text(texts[lo: lo + self.gpt.max_batch], self.device, refine[0])
                tokens += [i[i.less(self.tokenizer.break_0_ids)] for i in refined.ids]
                refined.destroy()
            texts, skip_refine_text = self.tokenizer.decode(tokens), True
            normalize = str  # the refined texts are spoken as they are
        if slots is None:
            slots = self.gpt.max_batch if split_text else max(2, min(self.gpt.max_batch, len(texts)))
        env = os.environ.get("CTB_DECODE_CHUNK")
        chunk = int(env) if env else 24 if split_text else min(p.stream_batch for p in params) if stream else 32
        out: queue.Queue = queue.Queue()  # (k, (chunk, last)), or (k, None) once text k's job has ended
        with self.gpt._open_slot_engine(ChatEngine, slots, cap, use_decoder, chunk, self, use_decoder,
                                        None if split_text else self.context,
                                        flags=_lib.engine_flags(dtype), prefill_budget=prefill_budget,
                                        kv_pool_bytes=kv_pool_bytes) as eng:
            subs = [eng._job(t, p, stream, skip_refine_text, r, split_text, max_split_batch, normalize, (out, k))
                    for k, (t, p, r) in enumerate(zip(texts, params, refine))]
            eng._enqueue(subs)
            jobs = [job for job, _ in subs]
            left = len(jobs)
            while left:
                if split_text and self.context.get():
                    eng.close(cancel=True)
                    self.logger.warning("generation is interrupted")
                    return
                stopped = eng._stopped  # read first: whatever the worker posted before it stopped is in `out` now
                try:
                    k, item = out.get(timeout=0.05)
                except queue.Empty:
                    if stopped:  # on an error, or on an interrupt it saw
                        eng.close()  # raises the worker's error, if it had one
                        self.logger.warning("generation is interrupted")
                        return
                    continue
                if item is None:  # job k ended: its result, or its error raised here
                    left -= 1
                    wav = jobs[k].result()
                    if not stream:
                        yield k, wav
                elif stream:
                    yield (k, *item)

    def _code_request(self, text, params, noise_batch=None):
        """The request ``_infer_code([text], ...)`` would decode as a batch of one (``noise_batch`` = (B, b): as row b
        of a batch of B)."""
        from .engine import Request

        temperature = params.temperature if isinstance(params.temperature, list) else [params.temperature] * self.config.gpt.num_vq
        num_code = self.config.gpt.num_audio_tokens - 1
        warpers, processors = gen_logits(num_code=num_code, top_P=params.top_P, top_K=params.top_K,
                                         repetition_penalty=params.repetition_penalty)
        return Request(emb=self._code_prompt(text, params), temperature=temperature, eos_token=num_code,
                       max_new_token=params.max_new_token, min_new_token=params.min_new_token,
                       logits_processors=(*processors, *warpers), manual_seed=params.manual_seed,
                       ensure_non_empty=params.ensure_non_empty, stream_batch=params.stream_batch,
                       noise_batch=noise_batch)

    def _code_prompt(self, text, params) -> torch.Tensor:
        """The speech-code prompt of one normalised ``text`` as ``_infer_code([text], ...)`` builds it for a batch of
        one: ``decorate_code_prompts`` with ``params.prompt`` / ``txt_smp`` / ``spk_emb``, the ``spk_smp`` codes, the
        embedding and ``Speaker.apply``; its valid positions ``[P, d]``."""
        input_ids, attention_mask, text_mask = self.tokenizer.encode(
            self.speaker.decorate_code_prompts([text], params.prompt, params.txt_smp, params.spk_emb),
            self.config.gpt.num_vq,
            prompt=(self.speaker.decode_prompt(params.spk_smp) if params.spk_smp is not None else None),
            device=self.device_gpt)
        emb = self.embed(input_ids, text_mask)
        if params.spk_emb is not None:
            self.speaker.apply(emb, params.spk_emb, input_ids, self.tokenizer.spk_emb_ids, self.gpt.device_gpt)
        valid = attention_mask[0].to(torch.bool).cpu()
        return emb[0][valid.to(emb.device)]

    def score(self, texts, codes, params_infer_code=None, lang=None, do_text_normalization=True,
              do_homophone_replacement=True, top_logprobs: int = 0) -> list:
        """The model's log-probability of given speech codes for each text: ``codes[i]`` (``[n, num_vq]`` ids, e.g.
        ``GenerationOutputs.ids``, or a recording's ``dvae.sample_audio(wav).T``) after the code prompt that
        ``infer`` builds for ``texts[i]`` with ``params_infer_code`` (``prompt``, ``txt_smp``, ``spk_smp``,
        ``spk_emb``; the normaliser as in ``infer``).  Returns per text an fp32 tensor ``[n, num_vq]`` of
        ``log softmax(z)[code]`` (``GPT.score``).  The quantity is defined at temperature 1 on the raw head logits, so
        the sampling fields of the params (temperature, top_P, top_K, repetition_penalty) do not enter.
        ``top_logprobs=N`` (1..20) makes each entry ``(lp, top_ids, top_lp)``: the codes the model expected most at
        every frame, ``[n, num_vq, N]``, and their log-probabilities (``GPT.score(top_logprobs=N)``)."""
        from .engine import check_top_logprobs

        check_top_logprobs(top_logprobs)
        texts = [texts] if isinstance(texts, str) else list(texts)
        params = params_infer_code or Chat.InferCodeParams()
        prompts = [self._code_prompt(self.normalizer(t, do_text_normalization, do_homophone_replacement, lang), params)
                   for t in texts]
        if top_logprobs:
            return self.gpt.score(prompts, list(codes), top_logprobs=top_logprobs)
        return self.gpt.score(prompts, list(codes))

    def _refine_request(self, text, params, noise_batch=None):
        """The text request ``_refine_text([text], ...)`` would generate as a batch of one (``noise_batch`` = (B, b): as
        row b of a batch of B)."""
        from .engine import Request

        input_ids, attention_mask, text_mask = self.tokenizer.encode(
            self.speaker.decorate_text_prompts([text], params.prompt), self.config.gpt.num_vq, device=self.device_gpt)
        warpers, processors = gen_logits(num_code=self.tokenizer.len, top_P=params.top_P, top_K=params.top_K,
                                         repetition_penalty=params.repetition_penalty)
        emb = self.embed(input_ids, text_mask)
        valid = attention_mask[0].to(torch.bool).cpu()
        return Request(emb=emb[0][valid.to(emb.device)], temperature=[params.temperature],
                       eos_token=self.tokenizer.eos_token, max_new_token=params.max_new_token,
                       min_new_token=params.min_new_token, logits_processors=(*processors, *warpers),
                       manual_seed=params.manual_seed, ensure_non_empty=params.ensure_non_empty, infer_text=True,
                       noise_batch=noise_batch)

    def _refined_text(self, out) -> str:
        """The text ``_infer`` makes of one refined row: ids below ``break_0_ids``, decoded."""
        ids = out.ids[0]
        return self.tokenizer.decode([ids[ids.less(self.tokenizer.break_0_ids)]])[0]

    def open_engine(self, slots: Optional[int] = None, max_new_cap: int = 2048, use_decoder: bool = True,
                    dtype=torch.float32, prefill_budget: Optional[int] = None, kv_pool_bytes: Optional[int] = None,
                    logprobs: bool = False, top_logprobs: int = 0):
        """A long-lived slot engine (``GPT.open_engine``) that synthesises texts submitted from any thread while it
        decodes: ``engine.submit(text, params_infer_code=None, stream=False, skip_refine_text=True, ...) -> Job``,
        ``Job.cancel()`` for one text, ``close(cancel=False)`` or a ``with`` block to drain it (``close(cancel=True)``
        is its interrupt; ``Chat.context`` is not read).  ``slots`` defaults to the handle's ``max_batch`` (up to 64
        for ``dtype=torch.float16``); every stage's ``max_new_token`` must be at most ``max_new_cap``, and its prompt
        plus ``max_new_token`` at most ``max_context`` (prompts over 1,024 tokens as in ``infer_continuous``).  See
        ``ChatEngine.submit``.  ``dtype`` as in
        ``infer_continuous``: every stage of every job runs on that engine.  ``prefill_budget`` (prompt columns per
        poll, at least 128; default None) bounds the prefill the running jobs wait for at each poll
        (``infer_continuous``); a job cancelled while its prompt is in progress frees its slot at the next poll.
        ``kv_pool_bytes`` (default None) bounds the engine's KV memory as in ``infer_continuous``; ``submit`` refuses
        a stage that does not fit in the pool alone.

        ``logprobs=True``: every finished job has ``Job.logprobs`` (CPU fp32), the log-probability of each speech
        token under the model's head logits at temperature 1 (``GPT.generate_continuous(logprobs=True)``): the
        ``[n, num_vq]`` tensor of its code request for a one-sentence job, a list of such tensors in take order with
        ``takes``, and in sentence order with ``split_text=True`` (neither the reference stage nor refinements are
        included).  The waveforms are the same as without it.  None on an engine opened without it.

        ``top_logprobs=N`` (1..20): every finished job also has ``Job.top_logprobs``, with the same structure: per code
        request a CPU pair ``(ids, lp)`` of ``[n, num_vq, N]`` tensors, the N codes with the largest head logits at
        each frame and their log-probabilities (``GPT.generate_continuous(top_logprobs=N)``).  Independent of
        ``logprobs``; the waveforms are the same as without it.  None on an engine opened without it."""
        from .engine import check_top_logprobs

        check_top_logprobs(top_logprobs)
        flags = _lib.engine_flags(dtype)
        check_prefill_budget(prefill_budget)
        assert self.has_loaded(use_decoder=use_decoder)
        return self.gpt._open_slot_engine(ChatEngine, self.gpt.max_batch if slots is None else slots, max_new_cap,
                                          use_decoder, None, self, use_decoder, flags=flags,
                                          prefill_budget=prefill_budget, kv_pool_bytes=kv_pool_bytes,
                                          logprobs=logprobs, top_logprobs=top_logprobs)

    def interrupt(self):
        self.context.set(True)

    # core.py:386-503
    def _infer(self, text, stream, lang, skip_refine_text, refine_text_only, use_decoder, do_text_normalization,
               do_homophone_replacement, split_text, max_split_batch, params_refine_text, params_infer_code):
        assert self.has_loaded(use_decoder=use_decoder)
        if not isinstance(text, list):
            text = [text]
        text = [self.normalizer(t, do_text_normalization, do_homophone_replacement, lang) for t in text]
        if not skip_refine_text:
            tokens = []
            for lo in range(0, len(text), self.gpt.max_batch):          # one batch in the reference; chunks beyond max_batch
                refined = self._refine_text(text[lo: lo + self.gpt.max_batch], self.device, params_refine_text)
                tokens += [i[i.less(self.tokenizer.break_0_ids)] for i in refined.ids]
                refined.destroy()
            text = self.tokenizer.decode(tokens)
            if refine_text_only:
                if split_text and isinstance(text, list):
                    text = "\n".join(text)
                yield text
                return
        if split_text and len(text) > 1 and params_infer_code.spk_smp is None:
            # core.py:435-453: sentence 0 is synthesised once on its own and its audio, re-encoded by the DVAE encode
            # branch, becomes the speaker prompt (spk_smp / txt_smp) of every sentence - this keeps one voice across them
            refer_text = text[0]
            result = next(self._infer_code(refer_text, False, self.device, use_decoder, params_infer_code))
            wavs = self._decode_to_wavs(result.hiddens if use_decoder else result.ids, use_decoder)
            result.destroy()
            assert len(wavs) == 1
            params_infer_code.spk_smp = self.sample_audio_speaker(wavs[0])
            params_infer_code.txt_smp = refer_text
        if stream:
            length, pass_batch_count = 0, 0
        if split_text:
            n = (len(text) + max_split_batch - 1) // max_split_batch
        else:
            # the reference runs all texts as one batch; batches beyond the handle's max_batch run as consecutive chunks
            # (rows are independent, so the result per text is the same; noise rows restart per chunk, SURVEY.md 8e)
            max_split_batch = min(len(text), self.gpt.max_batch)
            n = (len(text) + max_split_batch - 1) // max_split_batch
        for i in range(n):
            chunk = text[i * max_split_batch: (i + 1) * max_split_batch]
            for result in self._infer_code(chunk, stream, self.device, use_decoder, params_infer_code):
                res = result.hiddens if use_decoder else result.ids
                if stream:
                    # core.py:455-503 decodes the CUMULATIVE sequence at every yield and slices [length, length +
                    # stream_speed) out of it; the same samples are produced here from the token window they depend on
                    # (SURVEY.md 8f N2, decoder.decode_to_wavs_window)
                    pass_batch_count += 1
                    last = [r.clone() for r in res]
                    total = 512 * max(int(r.size(0)) for r in res) - 256
                    result.destroy()
                    if pass_batch_count <= params_infer_code.pass_first_n_batches:
                        continue
                    a, b = length, min(length + params_infer_code.stream_speed, total)
                    length = b
                    yield self._decode_window(last, use_decoder, a, b)
                else:
                    wavs = self._decode_to_wavs(res, use_decoder)
                    result.destroy()
                    yield wavs
            if stream:
                total = 512 * max(int(r.size(0)) for r in last) - 256
                new_wavs = self._decode_window(last, use_decoder, length, total)
                keep = np.sum(np.abs(new_wavs) > 1e-5, axis=0) > 0
                yield new_wavs[:][:, keep]

    # core.py:512-539 - hot path 2
    @torch.inference_mode()
    def _decode_to_wavs(self, result_list: List[torch.Tensor], use_decoder: bool):
        return decode_to_wavs(result_list, use_decoder, self.decoder, self.dvae)

    @torch.inference_mode()
    def _decode_window(self, result_list: List[torch.Tensor], use_decoder: bool, a: int, b: int) -> np.ndarray:
        """Samples [a, b) of ``_decode_to_wavs(result_list)`` from the tokens they depend on (streaming hand-off)."""
        return decode_to_wavs_window(result_list, use_decoder, self.decoder, self.dvae, a, b)

    def _vocos_decode(self, spec: torch.Tensor) -> np.ndarray:
        return self.vocos_engine().vocos_decode(spec).cpu().numpy()

    def vocos_engine(self):
        return self.decoder.engine

    # core.py:541-662 - hot path 1 (audio codes)
    @torch.no_grad()
    def _infer_code(self, text, stream: bool, device, return_hidden: bool, params):
        if not isinstance(text, list):
            text = [text]
        assert len(text), "text should not be empty"
        temperature = params.temperature if isinstance(params.temperature, list) else [params.temperature] * self.config.gpt.num_vq
        input_ids, attention_mask, text_mask = self.tokenizer.encode(
            self.speaker.decorate_code_prompts(text, params.prompt, params.txt_smp, params.spk_emb),
            self.config.gpt.num_vq,
            prompt=(self.speaker.decode_prompt(params.spk_smp) if params.spk_smp is not None else None),
            device=self.device_gpt)
        num_code = self.config.gpt.num_audio_tokens - 1
        warpers, processors = gen_logits(num_code=num_code, top_P=params.top_P, top_K=params.top_K,
                                         repetition_penalty=params.repetition_penalty)
        emb = self.embed(input_ids, text_mask)
        if params.spk_emb is not None:
            self.speaker.apply(emb, params.spk_emb, input_ids, self.tokenizer.spk_emb_ids, self.gpt.device_gpt)
        return self.gpt.generate(
            emb, input_ids, temperature=torch.tensor(temperature), eos_token=num_code, attention_mask=attention_mask,
            max_new_token=params.max_new_token, min_new_token=params.min_new_token,
            logits_processors=(*processors, *warpers), infer_text=False, return_hidden=return_hidden, stream=stream,
            show_tqdm=params.show_tqdm, ensure_non_empty=params.ensure_non_empty, stream_batch=params.stream_batch,
            manual_seed=params.manual_seed, context=self.context)

    # core.py:664-751 - hot path 1 (text refinement)
    @torch.no_grad()
    def _refine_text(self, text, device, params):
        if not isinstance(text, list):
            text = [text]
        input_ids, attention_mask, text_mask = self.tokenizer.encode(
            self.speaker.decorate_text_prompts(text, params.prompt), self.config.gpt.num_vq, device=self.device_gpt)
        warpers, processors = gen_logits(num_code=self.tokenizer.len, top_P=params.top_P, top_K=params.top_K,
                                         repetition_penalty=params.repetition_penalty)
        emb = self.embed(input_ids, text_mask)
        return next(self.gpt.generate(
            emb, input_ids, temperature=torch.tensor([params.temperature]), eos_token=self.tokenizer.eos_token,
            attention_mask=attention_mask, max_new_token=params.max_new_token, min_new_token=params.min_new_token,
            logits_processors=(*processors, *warpers), infer_text=True, stream=False, show_tqdm=params.show_tqdm,
            ensure_non_empty=params.ensure_non_empty, manual_seed=params.manual_seed, context=self.context))


class StreamWindows:
    """The streaming hand-off of ``Chat._infer`` (reference core.py:455-503) for one request decoded alone: turns its
    cumulative GPT yields into the sample windows ``infer([text], stream=True, split_text=False)`` yields.  The first
    ``pass_first_n_batches`` yields are skipped (and do not advance the position); every other yield, the final one
    included, takes the next ``stream_speed`` samples, clamped to the 512 n - 256 samples of its n tokens; the final
    yield is then followed by the rest of the sequence, whose all-silent samples are dropped."""

    def __init__(self, stream_speed: int, pass_first_n_batches: int):
        self.speed, self.skip = int(stream_speed), int(pass_first_n_batches)
        self.length = self.count = 0

    def windows(self, n_tokens: int, last: bool):
        """``[(a, b, flush)]``: the sample windows of one GPT yield of `n_tokens` tokens (b <= a: an empty chunk)."""
        if n_tokens == 0:  # a seeded request that ended empty: one empty closing chunk
            return [(0, 0, True)] if last else []
        total = 512 * n_tokens - 256
        out = []
        self.count += 1
        if self.count > self.skip:
            a, b = self.length, min(self.length + self.speed, total)
            self.length = b
            out.append((a, b, False))
        if last:
            out.append((self.length, total, True))
        return out


def _decode_windows(dev, jobs, model: DVAE, use_decoder: bool):
    """One poll's path-2 work on the slot engine ``dev``: ``jobs`` are ``(key, slot, n_tokens, a, b, flush, last)``,
    samples [a, b) of the decode of the slot's first ``n_tokens`` tokens (``flush``: drop its silent samples) ->
    ``[(key, chunk [1, m] float32, last)]`` in the same order.  Each window's token range (``decoder.stream_window``)
    is read straight from the engine's hidden states (``model`` = the DVAE decoder) or codes (``model`` = the code
    DVAE, ``use_decoder=False``); every non-empty window goes into one ``decode_rows`` call and is cut out of its
    row."""
    thr = np.float32(1e-5)
    buf = dev.hid_out if use_decoder else dev.ids_out
    due = [k for k, j in enumerate(jobs) if j[4] > j[3]]
    chunks: Dict[int, np.ndarray] = {}
    if due:
        rows, cuts = [], []
        for k in due:
            _, s, n, a, b = jobs[k][:5]
            a, b, t0, t1 = stream_window(n, a, b)
            # an interrupted request that was suspended: its image holds its tokens
            rows.append((s.row(use_decoder) if isinstance(s, SlotImage) else buf[s])[t0:t1])
            cuts.append((a - 512 * t0, b - 512 * t0))
        wavs = model.engine.decode_rows(rows, 1 if use_decoder else 2)
        flat = torch.cat([w[c0:c1] for w, (c0, c1) in zip(wavs, cuts)]).cpu().numpy()
        off = 0
        for k, (c0, c1) in zip(due, cuts):
            chunks[k] = flat[None, off: off + c1 - c0]
            off += c1 - c0
    out = []
    for k, (i, _, _, _, _, flush, last) in enumerate(jobs):
        chunk = chunks.get(k, np.zeros((1, 0), dtype=np.float32))
        if flush:
            chunk = chunk[:, np.abs(chunk[0]) > thr]
        out.append((i, chunk, last))
    return out


class _Paragraph:
    """A job's state on ``ChatEngine`` (a text without ``split_text`` is a paragraph of one sentence): its reference
    stage, which request speaks which sentence, and the in-order assembly of the sentences' audio (``add``).  ``sink`` =
    (queue, key): the chunks and the end of the job are also posted there, for ``Chat.infer_continuous*``.  ``split``:
    the job was submitted with ``split_text=True``."""

    def __init__(self, n: int, stream_params, sink=None, takes: bool = False, split: bool = False):
        self.n, self.sink, self.takes, self.split = n, sink, takes, split
        self.logprobs: Optional[list] = None  # an engine with logprobs: each sentence's, once its code request ends
        self.top_logprobs: Optional[list] = None  # an engine with top_logprobs: each sentence's (ids, lp), likewise
        self.windows = ([StreamWindows(stream_params.stream_speed, stream_params.pass_first_n_batches)
                         for _ in range(n)] if stream_params is not None else None)
        self.ref = None
        self.order: Dict[object, int] = {}  # Request -> sentence number
        self.job: Optional[Job] = None
        self.parts: List[list] = [[] for _ in range(n)]
        self.closed = [False] * n
        self.next = 0  # the first sentence whose audio is not all out
        self._ended = False

    def add(self, k: int, chunk: np.ndarray, last: bool) -> None:
        """Sentence k's next chunk (its whole stripped waveform when not streaming); ``last``: its final one."""
        self.parts[k].append(chunk)
        self.closed[k] = self.closed[k] or last
        out = []
        while self.next < self.n:
            if self.windows is not None:
                out += self.parts[self.next]
                self.parts[self.next] = []
            if not self.closed[self.next]:
                break
            self.next += 1
        done = self.next == self.n
        job = self.job
        if done and self.logprobs is not None:
            job.logprobs = self.logprobs if self.takes or self.split else self.logprobs[0]
        if done and self.top_logprobs is not None:
            job.top_logprobs = self.top_logprobs if self.takes or self.split else self.top_logprobs[0]
        if self.windows is not None:
            for j, c in enumerate(out):
                item = (c, done and j == len(out) - 1)
                job._put(item)
                if self.sink is not None:
                    self.sink[0].put((self.sink[1], item))
            if done:
                job._finish(None)
        elif done and self.takes:  # n takes of one sentence: one waveform each
            job._finish([np.concatenate([c[0] for c in part]) for part in self.parts])
        elif done:
            job._finish(np.concatenate([c[0] for part in self.parts for c in part]))
        if done:
            self.ended()

    def ended(self) -> None:
        if self.sink is not None and not self._ended:
            self.sink[0].put((self.sink[1], None))
        self._ended = True


class _SpeakerSampler:
    """``Request.prepare`` of the paragraphs' reference stages on one engine: the whole sequences of the reference stages
    that end at a poll are decoded in one ``decode_rows`` call, straight from the engine's buffers, and the waveforms
    are read in place by one ``encode_rows`` call; ``take`` hands each stage's speaker-prompt string to its ``then``."""

    def __init__(self, chat: "Chat", model: DVAE, use_decoder: bool):
        self.chat, self.model, self.use_decoder = chat, model, use_decoder
        self._out: Dict[object, object] = {}

    def __call__(self, dev, items) -> None:
        rows = []
        for r, s, n in items:
            if n == 0:  # infer() gets no reference waveform from a seeded sentence 0 that ends empty
                self._out[r] = RuntimeError("sentence 0 of the paragraph ended empty: there is no audio to sample a "
                                            "speaker from")
            elif 512 * n - 256 <= ENC_NFFT // 2:
                self._out[r] = _lib.CtbError(f"reflect padding needs more than {ENC_NFFT // 2} samples (sentence 0 "
                                             f"of the paragraph has {n} token)")
            else:
                rows.append((r, s, n))
        if not rows:
            return
        buf = dev.hid_out if self.use_decoder else dev.ids_out
        wavs = self.model.engine.decode_rows([buf[s, :n] for _, s, n in rows], 1 if self.use_decoder else 2)
        codes = self.chat.dvae.audio_encoder.encode_rows(wavs)
        for (r, _, _), c in zip(rows, codes):
            self._out[r] = self.chat.speaker.encode_prompt(c)

    def take(self, r):
        v = self._out.pop(r)
        if isinstance(v, BaseException):
            raise v
        return v


class _RefineGraph:
    """The stage graph of a refined paragraph (``ChatEngine.submit(split_text=True, skip_refine_text=False)``).

    Each of the n sentences is refined by a text request of its own, whose ``then`` is ``then(k)``; ``refined[k]`` is
    its text once it has ended (``refined_text(outputs)``).  With a reference stage (``reference`` given: n > 1 and no
    ``spk_smp``), refinement 0's follow-up is ``reference(r_0)``, the code request of the refined sentence 0 alone,
    and the reference stage's ``then`` takes the speaker sample with ``sample(request)``.  Sentence k's code request,
    ``code(k, r_k, (spk_smp, txt_smp) or None)``, needs both ``r_k`` and the sample, and is made exactly once, by
    whichever of the two stages ends last (the join): refinement k's ``then`` returns it when the sample is known and
    None otherwise, and the reference stage's ``then`` returns the code requests of every sentence refined by then, in
    sentence order.  Without a reference stage each refinement's ``then`` returns its code request.  A refinement that
    ended empty raises in its ``then``, which fails the job, as a seeded first-step EOS makes ``infer`` raise; with
    ``speak_empty`` (a text submitted without ``split_text``) the empty refined text is spoken instead."""

    def __init__(self, n: int, refined_text, code, reference=None, sample=None, speak_empty=False):
        self.n, self.refined_text, self.code, self.reference, self.sample = n, refined_text, code, reference, sample
        self.speak_empty = speak_empty
        self.refined: List[Optional[str]] = [None] * n
        self.ref = None  # the reference stage's request, once refinement 0 has ended
        self.spk = None  # (spk_smp, txt_smp), once the reference stage has ended
        self._made = [False] * n

    def then(self, k: int):
        def then(out):
            if int(out.ids[0].shape[0]) == 0 and not self.speak_empty:
                raise RuntimeError(f"the refinement of sentence {k} of the paragraph ended empty")
            self.refined[k] = self.refined_text(out)
            if self.reference is None:
                return self._make(k)
            if k == 0:
                self.ref = self.reference(self.refined[0])
                self.ref.then = self._reference_then
                return self.ref
            return self._make(k) if self.spk is not None else None
        return then

    def _reference_then(self, out):
        self.spk = (self.sample(self.ref), self.refined[0])
        return [self._make(k) for k in range(self.n) if self.refined[k] is not None]

    def _make(self, k: int):
        assert not self._made[k], f"sentence {k}'s code request was made twice"
        self._made[k] = True
        return self.code(k, self.refined[k], self.spk)


class ChatEngine(OpenEngine):
    """``Chat.open_engine``: an open slot engine whose jobs are texts (see there).  At each poll every window due for a
    streaming job and the whole sequence of every non-streaming job that completed go into one ``decode_rows`` call."""

    def __init__(self, make_device, chunk, check, device, on_close, chat: "Chat", use_decoder: bool, context=None,
                 max_new_cap: Optional[int] = None, prefill_budget: Optional[int] = None, slots: Optional[int] = None):
        self.chat, self.use_decoder = chat, use_decoder
        self.model = chat.decoder if use_decoder else chat.dvae
        self._sampler = _SpeakerSampler(chat, self.model, use_decoder)
        super().__init__(make_device, chunk, check, device, on_close, max_new_cap, context, prefill_budget, slots)

    def submit(self, text: str, params_infer_code=None, stream=False, skip_refine_text=True, params_refine_text=None,
               lang=None, do_text_normalization=True, do_homophone_replacement=True, split_text=False,
               max_split_batch=1, takes: int = 1) -> Job:
        """Queue one text -> ``Job``: ``result()`` is the waveform ``infer_continuous`` yields for it, or with
        ``stream=True`` the job iterates the ``(chunk, last)`` pairs ``infer_continuous_stream`` yields for it.
        ``skip_refine_text=False`` refines the text on the engine first (``refine_on_engine=True``).  A cancelled
        job's ``result()`` raises ``concurrent.futures.CancelledError`` and its stream ends.

        ``split_text=True``: the text is a paragraph, split into sentences by ``infer``'s rule (``split_sentences``),
        and keeps one voice across them as ``infer`` does.  With one sentence, or with an explicit ``spk_smp``, each
        sentence is one request with these params.  Otherwise sentence 0 first runs once alone (the reference stage);
        its whole, unstripped waveform is encoded by the DVAE encode branch into the speaker sample ``spk_smp``
        (``Job.spk_smp`` once known), with ``txt_smp`` = sentence 0, and every sentence, sentence 0 included, is then
        a request of its own with a copy of the params carrying them.  The reference stages ending at one poll are
        decoded in one ``decode_rows`` call and encoded in one ``encode_rows`` call.  ``result()`` is the sentences'
        waveforms, each silence-stripped, concatenated in order: what ``infer(text, split_text=True,
        max_split_batch=1, skip_refine_text=True)[0]`` returns (the caller's params are not modified here, while
        ``infer`` stores the sample on them).  Streamed, the chunks are each sentence's chunks in sentence order,
        those of ``infer([sentence], stream=True, split_text=False)`` with the sample on its params; a later
        sentence's chunks are held until the earlier one's final chunk is out, and ``last`` marks only the final
        chunk of the last sentence.  Unlike ``infer(stream=True)``, whose stream position runs on across its batches,
        each sentence's stream starts at its own first sample.  A reference stage too short to encode or that ended
        empty, or a sentence whose prompt breaks the engine's limits, fails that job only; its other live stages are
        cancelled at the next poll.

        ``max_split_batch`` = m: sentence k samples as row ``k mod m`` of ``infer``'s code batch of
        ``min(m, n - m * (k // m))`` sentences (``Request.noise_batch``), so a seeded paragraph is what ``infer(...,
        max_split_batch=m)`` returns; the default 1 is the batch of one of each sentence.

        ``skip_refine_text=False`` with ``split_text=True`` refines every sentence on the engine first, each as row
        ``k mod max_batch`` of ``infer``'s refinement batch, with ``params_refine_text``; ``Job.refined`` lists the
        refined sentences as they end.  The reference stage speaks the refined sentence 0, and each sentence's code
        request starts as soon as both its refinement and the speaker sample are done (see ``_RefineGraph``).
        ``result()`` is then what ``infer(text, use_decoder=False, max_split_batch=m, params_refine_text=...)[0]``
        returns, bit for bit on the code path when seeded (with the default arguments and m = 4: ``infer(text)``).
        A refinement that ends empty fails the job, as it makes ``infer`` raise.  Without ``split_text`` the text is
        a paragraph of one sentence, and a refinement that ends empty goes on to speak the empty refined text.

        ``takes`` = n > 1: n takes of the text, to keep the best (ChatTTS output varies from seed to seed).
        ``result()`` is the list of their n waveforms, each what a one-sentence job gives; ``Job.cancel()`` cancels
        every take.  The takes are n code requests of one ``Request.prompt_key``: once one of them runs, the others
        share its prompt's KV and prefill only the last chunk of at most 128 columns, with the same results.  With
        ``manual_seed`` set, take k samples as row k of ``infer([text] * n)``'s code batch (``noise_batch`` = (n, k));
        without it, each take draws its own seed.  It takes ``stream=False``, ``split_text=False`` and
        ``skip_refine_text=True``, and n at most the engine's slots and the handle's ``max_batch``."""

        def normalize(t):
            return self.chat.normalizer(t, do_text_normalization, do_homophone_replacement, lang)

        if takes != 1:
            job, requests = self._takes_job(text, params_infer_code or Chat.InferCodeParams(), takes, stream,
                                            skip_refine_text, split_text, normalize)
            self._enqueue([(job, requests)])
            return job

        job, requests = self._job(text, params_infer_code or Chat.InferCodeParams(), stream, skip_refine_text,
                                  params_refine_text or Chat.RefineTextParams(), split_text, max_split_batch, normalize)
        self._enqueue([(job, requests)])
        return job

    def _takes_job(self, text, params, takes, stream, skip_refine_text, split_text, normalize):
        """``submit``'s job of ``takes`` takes of ``text`` and its requests -> ``(Job, requests)``."""
        n = int(takes)
        if n != takes or n < 1:
            raise ValueError(f"takes={takes!r}: a positive int")
        if stream or split_text or not skip_refine_text:
            raise ValueError("takes > 1 needs stream=False, split_text=False and skip_refine_text=True")
        limit = min(self.chat.gpt.max_batch, self.slots or self.chat.gpt.max_batch)
        if n > limit:
            raise ValueError(f"takes={n} exceed this engine's slots and the handle's max_batch ({limit})")
        if self.max_new_cap is not None and params.max_new_token > self.max_new_cap:
            raise ValueError(f"max_new_token {params.max_new_token} exceeds max_new_cap={self.max_new_cap}")
        first = self.chat._code_request(normalize(text), params)
        key = object()  # this job's takes, and nothing else, share a prompt
        seeded = params.manual_seed is not None
        para = _Paragraph(n, None, takes=True)
        reqs = []
        for k in range(n):
            r = replace(first, noise_batch=(n, k) if seeded else None, prompt_key=key)
            para.order[r] = k
            reqs.append(r)
        para.job = self._new_job(reqs, False, para)
        return para.job, reqs

    def _job(self, text, params, stream, skip_refine_text, refine, split_text, max_split_batch, normalize, sink=None):
        """``submit``'s job, not queued yet, and its first requests -> ``(Job, requests)``; ``normalize`` maps each
        sentence to the text it speaks, ``sink`` as in ``_Paragraph``."""
        chat = self.chat
        if self.max_new_cap is not None and params.max_new_token > self.max_new_cap:
            # a speech stage made by a follow-up is only checked when it is made: check the limit here, in the caller's
            # thread
            raise ValueError(f"max_new_token {params.max_new_token} exceeds max_new_cap={self.max_new_cap}")
        m = int(max_split_batch)
        if m < 1:
            raise ValueError("max_split_batch must be >= 1")
        # the prompts are embedded here, on the caller's stream: ctb_gpt_embed_prompt is the one handle call that may
        # run beside the worker (it only reads the weights); _enqueue orders the engine's stream after the caller's
        sentences = [normalize(t) for t in (split_sentences(text) if split_text else [text])]
        if not sentences:
            raise ValueError("split_text=True: the text has no sentence")
        n = len(sentences)
        if min(m, n) > chat.gpt.max_batch:
            raise ValueError(f"max_split_batch={m}: a batch of {min(m, n)} sentences exceeds this handle's "
                             f"max_batch={chat.gpt.max_batch}")
        para = _Paragraph(n, params if stream else None, sink, split=split_text)
        spk_stage = n > 1 and params.spk_smp is None
        if spk_stage and chat.dvae.audio_encoder is None:
            raise RuntimeError("this DVAE checkpoint carries no encoder / VQ weights: cannot sample a speaker")

        def code(k, t, sample):  # sentence k's request: a copy of the params carrying the sample, row k mod m
            p = copy.copy(params)
            if sample is not None:
                p.spk_smp, p.txt_smp = sample
            r = chat._code_request(t, p, noise_batch=(min(m, n - m * (k // m)), k % m))
            para.order[r] = k
            return r

        def reference(t):  # the reference stage: sentence 0 alone, as infer() synthesises it
            para.ref = chat._code_request(t, copy.copy(params))
            para.ref.prepare = self._sampler
            return para.ref

        def sample(ref):
            spk = self._sampler.take(ref)
            para.job.spk_smp = spk
            return spk

        if not skip_refine_text:
            B = chat.gpt.max_batch  # infer() refines a paragraph's sentences in batches of up to max_batch
            graph = _RefineGraph(n, chat._refined_text, code, reference if spk_stage else None,
                                 sample if spk_stage else None, speak_empty=not split_text)
            reqs = []
            for k, t in enumerate(sentences):
                r = chat._refine_request(t, refine, noise_batch=(min(B, n - B * (k // B)), k % B))
                r.then = graph.then(k)
                r.stream_batch = params.stream_batch  # the engine polls at the smallest stream_batch of its requests
                reqs.append(r)
        elif not spk_stage:
            reqs = [code(k, t, None) for k, t in enumerate(sentences)]
        else:
            ref = reqs = reference(sentences[0])

            def then(out):
                smp = (sample(ref), sentences[0])
                return [code(k, t, smp) for k, t in enumerate(sentences)]

            ref.then = then
        para.job = self._new_job(reqs, stream, para)
        if not skip_refine_text:
            para.job.refined = graph.refined
        return para.job, reqs

    def _serve(self, dev, requests, batch, jobs) -> None:
        wjobs = []  # ((paragraph, sentence), slot, n_tokens, a, b, flush, last)
        for (i, s, n, last), (job, final) in zip(batch, jobs):
            para = job.state
            if i in self.stats.failed:
                job._fail(self.stats.failed[i])
                para.ended()
            elif job.done():
                continue
            elif i in self.stats.cancelled:
                job._stop()
                para.ended()
            elif requests[i].infer_text or requests[i] is para.ref:
                continue  # a refinement, or the reference stage, whose audio only becomes the speaker sample
            else:
                k = para.order[requests[i]]
                lp_on = getattr(dev, "lp_out", None) is not None  # an engine opened with logprobs
                top_on = getattr(dev, "top_ids_out", None) is not None  # with top_logprobs
                if last and (lp_on or top_on):
                    out = dev.empty(i) if s is None else dev.harvest(s, n, copy=False)
                    if lp_on:
                        if para.logprobs is None:
                            para.logprobs = [None] * para.n
                        para.logprobs[k] = out.logprobs[0].cpu()
                    if top_on:
                        if para.top_logprobs is None:
                            para.top_logprobs = [None] * para.n
                        para.top_logprobs[k] = tuple(t.cpu() for t in out.top_logprobs[0])
                if para.windows is not None:
                    ws = para.windows[k].windows(n, last)
                    wjobs += [((para, k), s, n, a, b, flush, last and j == len(ws) - 1) for j, (a, b, flush) in
                              enumerate(ws)]
                elif last:  # the whole sequence, silent samples dropped
                    wjobs.append(((para, k), s, n, 0, 512 * n - 256, True, True))
        for (para, k), chunk, last in _decode_windows(dev, wjobs, self.model, self.use_decoder):
            para.add(k, chunk, last)
