"""``Generator`` mixin: HF-style ``generate`` for LiBai models.

Spec: reference libai/inference/generator/generation_utils.py — input preparation (:58-230), cache/mask updates
(:232-271), warper / processor / stopping-criteria assembly (:273-405), ``greedy_search`` (:451-542),
``multinomial_sample`` (:544-643), ``beam_search`` (:645-785), ``generate`` (:787-1069).

Model contract (same as the reference): ``self.cfg`` provides the defaults (``bos/eos/pad_token_id``,
``max_length``, ``num_beams``, ``is_encoder_decoder``, ``use_cache`` …); ``forward(**inputs)`` returns a dict with
``"logits"`` (or ``"prediction_scores"``) ``[b, s, V]``; the model keeps its own KV cache (``past_key_values``,
``set_cache``) and may override ``prepare_inputs_for_generation`` / ``_reorder_cache``.  Under tensor parallelism
every rank runs the same search; sampled tokens are broadcast from rank 0 so the ranks cannot diverge.
"""
from __future__ import annotations

import contextlib
import inspect
import logging
import warnings
from typing import Callable, Dict, Iterable, List, Optional, Tuple, Union

import torch

from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dutil
import torch.distributed as dist

from .. import decode_graph
from ..kv_cache import KVCacheOwner, PagedKVCache, StaticKVCache
from .generation_beam_search import BeamScorer, BeamSearchScorer
from .generation_logits_processor import (
    EncoderNoRepeatNGramLogitsProcessor,
    ExponentialDecayLengthPenalty,
    ForcedBOSTokenLogitsProcessor,
    ForcedEOSTokenLogitsProcessor,
    HammingDiversityLogitsProcessor,
    InfNanRemoveLogitsProcessor,
    LogitsProcessorList,
    MinLengthLogitsProcessor,
    NoRepeatNGramLogitsProcessor,
    NormalizationLogitsProcessor,
    PrefixConstrainedLogitsProcessor,
    RepetitionPenaltyLogitsProcessor,
    TemperatureLogitsWarper,
    TopKLogitsWarper,
    TopPLogitsWarper,
    TypicalLogitsWarper,
)
from .generation_stopping_criteria import (
    MaxLengthCriteria,
    MaxTimeCriteria,
    StoppingCriteriaList,
    validate_stopping_criteria,
)

logger = logging.getLogger(__name__)

_DEFAULTS = dict(
    is_encoder_decoder=False, max_length=20, min_length=0, do_sample=False, early_stopping=False, num_beams=1,
    num_beam_groups=1, diversity_penalty=0.0, temperature=1.0, top_k=50, top_p=1.0, typical_p=1.0,
    repetition_penalty=1.0, length_penalty=1.0, no_repeat_ngram_size=0, encoder_no_repeat_ngram_size=0,
    num_return_sequences=1, output_scores=False, use_cache=True, bos_token_id=None, eos_token_id=None,
    pad_token_id=None, decoder_start_token_id=None, forced_bos_token_id=None, forced_eos_token_id=None,
    remove_invalid_values=False, exponential_decay_length_penalty=None, chunk_size_feed_forward=0,
    kv_cache_dtype=None, decode_graphs=False, assistant_model=None, num_assistant_tokens=None,
    prompt_lookup_num_tokens=None, max_matching_ngram_size=None, paged_kv_cache=False, prefix_cache_tokens=0,
)
# generate()'s arguments for the logits processors speculative decoding refuses, by processor
_PROCESSOR_ARGS = {
    HammingDiversityLogitsProcessor: "diversity_penalty", RepetitionPenaltyLogitsProcessor: "repetition_penalty",
    NoRepeatNGramLogitsProcessor: "no_repeat_ngram_size", EncoderNoRepeatNGramLogitsProcessor: "encoder_no_repeat_ngram_size",
    MinLengthLogitsProcessor: "min_length", PrefixConstrainedLogitsProcessor: "prefix_allowed_tokens_fn",
    ForcedBOSTokenLogitsProcessor: "forced_bos_token_id", ForcedEOSTokenLogitsProcessor: "forced_eos_token_id",
    InfNanRemoveLogitsProcessor: "remove_invalid_values", ExponentialDecayLengthPenalty: "exponential_decay_length_penalty",
    NormalizationLogitsProcessor: "renormalize_logits",
}
MAX_SPECULATIVE_TOKENS = 15   # k: a verify step of k + 1 tokens stays within the split-KV decode kernel's 16


def _kv_cache_dtype(value):
    """``generate(kv_cache_dtype=...)``: None (the weights' dtype), or ``"fp8"`` / ``torch.float8_e4m3fn``."""
    if value is None or value == torch.float8_e4m3fn:
        return value
    if isinstance(value, str) and value.lower() == "fp8":
        return torch.float8_e4m3fn
    raise ValueError(f"kv_cache_dtype must be None, 'fp8' or torch.float8_e4m3fn, got {value!r}")


def prompt_lookup(seq: List[int], k: int, max_ngram: int) -> List[int]:
    """Prompt-lookup proposals for one sample (HF's rule): for n from ``max_ngram`` down to 1, the earliest earlier
    occurrence of the last n tokens of ``seq`` that has at least one following token; up to ``k`` of the tokens that
    follow it, padded to ``k`` by repeating the last one (the last token of ``seq`` when nothing matches).  The filler
    only costs acceptance: greedy acceptance keeps only tokens the target chooses itself."""
    L = len(seq)
    out: List[int] = []
    for n in range(min(max_ngram, L - 1), 0, -1):
        tail = seq[L - n :]
        for i in range(L - n):   # i + n < L: the occurrence has a following token
            if seq[i : i + n] == tail:
                out = seq[i + n : i + n + k]
                break
        if out:
            break
    fill = out[-1] if out else seq[-1]
    return out + [fill] * (k - len(out))


def _decode_graphs(value) -> bool:
    """``generate(decode_graphs=...)``: a bool."""
    if not isinstance(value, bool):
        raise ValueError(f"decode_graphs must be True or False, got {value!r}")
    return value


def _paged_kv_cache(value) -> bool:
    """``generate(paged_kv_cache=...)``: a bool."""
    if not isinstance(value, bool):
        raise ValueError(f"paged_kv_cache must be True or False, got {value!r}")
    return value


def _prefix_cache_tokens(value) -> int:
    """``generate(prefix_cache_tokens=...)``: an int >= 0."""
    if isinstance(value, bool) or not isinstance(value, int) or value < 0:
        raise ValueError(f"prefix_cache_tokens must be an int >= 0, got {value!r}")
    return value


@contextlib.contextmanager
def _call_state(model, kv_cache_dtype, decode_graphs: bool, paging=None):
    """A model's state for one ``generate()`` call, restored when it ends: eval mode, the call's cache format when it
    gives one (``allocate_kv_cache`` reads it: ``kv_cache_dtype``, and ``paging`` = (sequences per prompt, prompt
    length) for a paged cache) and, with ``decode_graphs``, its decode graphs."""
    was_training, saved_kv_cache_dtype = model.training, getattr(model, "kv_cache_dtype", None)
    model.eval()
    try:
        if kv_cache_dtype is not None:
            model.kv_cache_dtype = kv_cache_dtype
        if decode_graphs:
            model._decode_graphs = decode_graph.DecodeCall()
        if paging is not None:
            model.kv_cache_paging = paging
        yield
    finally:
        model.train(was_training)
        if kv_cache_dtype is not None:
            model.kv_cache_dtype = saved_kv_cache_dtype
        if decode_graphs:
            del model._decode_graphs   # back to the class's None
        if paging is not None:
            del model.kv_cache_paging


class Generator:
    # ------------------------------------------------------------------ configuration access
    def _gcfg(self, key):
        cfg = getattr(self, "cfg", None)
        if cfg is not None:
            try:
                value = cfg.get(key, None) if hasattr(cfg, "get") else getattr(cfg, key, None)
            except Exception:
                value = None
            if value is not None:
                return value
        return _DEFAULTS[key]

    def _pick(self, value, key):
        return value if value is not None else self._gcfg(key)

    def _device(self):
        # parameters owned by other pipeline stages are `meta` placeholders
        for p in self.parameters():
            if p.device.type != "meta":
                return p.device
        return dutil.get_dist_util().device

    # ------------------------------------------------------------------ input preparation
    def _prepare_model_inputs(self, inputs=None, bos_token_id=None, model_kwargs=None):
        input_name = "encoder_input_ids" if self._gcfg("is_encoder_decoder") else "input_ids"
        model_kwargs = {k: v for k, v in model_kwargs.items() if v is not None or k != input_name}
        inputs_kwarg = model_kwargs.pop(input_name, None)
        if inputs_kwarg is not None and inputs is not None:
            raise ValueError(
                f"`inputs` were passed alongside {input_name} which is not allowed. "
                f"Make sure to either pass inputs or {input_name}=..."
            )
        if inputs_kwarg is not None:
            inputs = inputs_kwarg
        if inputs is None:
            inputs = self._prepare_input_ids_for_generation(bos_token_id, model_kwargs.get("encoder_outputs"))
        return inputs, input_name, model_kwargs

    def prepare_inputs_for_generation(self, input_ids, **kwargs):
        """Override for model-specific step inputs (cache-aware slicing, masks…)."""
        return {"input_ids": input_ids}

    def _prepare_input_ids_for_generation(self, bos_token_id, encoder_outputs):
        if self._gcfg("is_encoder_decoder") and encoder_outputs is not None:
            return torch.full(encoder_outputs.shape[:-1], -100, dtype=torch.long, device=encoder_outputs.device)
        if bos_token_id is None:
            raise ValueError("`bos_token_id` has to be defined when no `input_ids` are provided.")
        return torch.full((1, 1), bos_token_id, dtype=torch.long, device=self._device())

    def _prepare_attention_mask_for_generation(self, inputs, pad_token_id, eos_token_id):
        is_input_ids = inputs.dim() == 2 and inputs.dtype in (torch.int32, torch.int64)
        has_pad = pad_token_id is not None and bool((inputs == pad_token_id).any())
        pad_is_not_eos = eos_token_id is None or pad_token_id != eos_token_id
        if is_input_ids and has_pad and pad_is_not_eos:
            return inputs.ne(pad_token_id)
        return torch.ones(inputs.shape[:2], dtype=torch.bool, device=inputs.device)

    def _prepare_encoder_decoder_kwargs_for_generation(self, inputs_tensor, model_kwargs, model_input_name):
        """Encoder-decoder models keep the encoder states in their own cache (``set_cache``): the encoder runs
        inside the first decoding step, so only the inputs are recorded here."""
        model_kwargs[model_input_name] = inputs_tensor
        if "encoder_decoder_attn_mask" in inspect.signature(self.forward).parameters:
            model_kwargs.setdefault("encoder_decoder_attn_mask", model_kwargs.get("encoder_attn_mask"))
        return model_kwargs

    def _prepare_decoder_input_ids_for_generation(self, batch_size, decoder_start_token_id=None, bos_token_id=None,
                                                  model_kwargs=None):
        if model_kwargs is not None and "decoder_input_ids" in model_kwargs:
            return model_kwargs.pop("decoder_input_ids")
        start = self._get_decoder_start_token_id(decoder_start_token_id, bos_token_id)
        return torch.full((batch_size, 1), start, dtype=torch.long, device=self._device())

    def _get_decoder_start_token_id(self, decoder_start_token_id=None, bos_token_id=None):
        if decoder_start_token_id is not None:
            return decoder_start_token_id
        if self._gcfg("is_encoder_decoder") and self._gcfg("decoder_start_token_id") is not None:
            return self._gcfg("decoder_start_token_id")
        if bos_token_id is not None:
            return bos_token_id
        if self._gcfg("bos_token_id") is not None:
            return self._gcfg("bos_token_id")
        raise ValueError("`decoder_start_token_id` or `bos_token_id` has to be defined for encoder-decoder generation.")

    @staticmethod
    def _expand_inputs_for_generation(input_ids, expand_size=1, is_encoder_decoder=False, attention_mask=None,
                                      encoder_outputs=None, **model_kwargs):
        idx = torch.arange(input_ids.shape[0], device=input_ids.device).view(-1, 1).repeat(1, expand_size).view(-1)
        input_ids = input_ids.index_select(0, idx)
        if attention_mask is not None:
            model_kwargs["attention_mask"] = attention_mask.index_select(0, idx)
        if is_encoder_decoder:
            for key in ("encoder_input_ids", "encoder_attn_mask", "encoder_decoder_attn_mask", "encoder_outputs"):
                value = encoder_outputs if key == "encoder_outputs" else model_kwargs.get(key)
                if value is not None:
                    model_kwargs[key] = value.index_select(0, idx.to(value.device))
        return input_ids, model_kwargs

    def _update_model_kwargs_for_generation(self, outputs, model_kwargs, is_encoder_decoder=False):
        if isinstance(outputs, dict) and "past_key_values" in outputs:
            model_kwargs["past"] = outputs["past_key_values"]
        else:
            past = getattr(self, "past_key_values", None)
            if isinstance(past, StaticKVCache):
                cached = past.length > 0   # the host mirror: valid on stages that own no layer, too
            else:
                # under pipeline parallelism a rank only holds the caches of its own layers (possibly none at all): the
                # model's `past_length` says whether a cache exists somewhere
                cached = bool(past) and (any(p is not None for p in past) or (
                    dutil.get_dist_util().pipeline_parallel_size > 1 and getattr(self, "past_length", 0) > 0))
            model_kwargs["past"] = past if cached else None
        key = "decoder_attn_mask" if is_encoder_decoder else "attention_mask"
        if model_kwargs.get(key) is not None:
            mask = model_kwargs[key]
            model_kwargs[key] = torch.cat([mask, mask.new_ones((mask.shape[0], 1))], dim=-1)
        return model_kwargs

    def _reorder_cache(self, past, beam_idx):
        """Default: every cached tensor is batch-major; models with another layout override this.  A
        :class:`StaticKVCache` is gathered in place."""
        if past is None:
            return None
        if isinstance(past, StaticKVCache):
            past.reorder_(beam_idx)
            return past

        def reorder(x):
            if torch.is_tensor(x):
                return x.index_select(0, beam_idx.to(x.device))
            if isinstance(x, (list, tuple)):
                return type(x)(reorder(y) for y in x)
            return x

        return reorder(past)

    def _apply_reordered_cache(self, past):
        """Write a reordered cache back into the model (models own their cache)."""
        if past is None:
            return
        if hasattr(self, "set_cache"):
            params = inspect.signature(self.set_cache).parameters
            if "encoder_states" in params:
                enc = getattr(self, "encoder_states", None)
                if enc is None and hasattr(self, "t5_model"):
                    enc = getattr(self.t5_model, "encoder_states", None)
                self.set_cache(enc, past)
            else:
                self.set_cache(past)
        else:
            self.past_key_values = past

    def _reset_cache(self):
        if hasattr(self, "set_cache"):
            params = inspect.signature(self.set_cache).parameters
            if "encoder_states" in params:
                self.set_cache(None, None)
            else:
                self.set_cache(None)
        elif hasattr(self, "past_key_values"):
            self.past_key_values = [None] * len(self.past_key_values)

    # ------------------------------------------------------------------ processors
    def _get_logits_warper(self, top_k=None, top_p=None, typical_p=None, temperature=None, num_beams=None,
                           renormalize_logits=None):
        top_k, top_p = self._pick(top_k, "top_k"), self._pick(top_p, "top_p")
        typical_p, temperature = self._pick(typical_p, "typical_p"), self._pick(temperature, "temperature")
        warpers = LogitsProcessorList()
        keep = 2 if (num_beams or 1) > 1 else 1
        if temperature is not None and temperature != 1.0:
            warpers.append(TemperatureLogitsWarper(float(temperature)))
        if top_k is not None and top_k != 0:
            warpers.append(TopKLogitsWarper(top_k=int(top_k), min_tokens_to_keep=keep))
        if top_p is not None and top_p < 1.0:
            warpers.append(TopPLogitsWarper(top_p=top_p, min_tokens_to_keep=keep))
        if typical_p is not None and typical_p < 1.0:
            warpers.append(TypicalLogitsWarper(mass=typical_p, min_tokens_to_keep=keep))
        if renormalize_logits:
            warpers.append(NormalizationLogitsProcessor())
        return warpers

    def _get_logits_processor(self, repetition_penalty, no_repeat_ngram_size, encoder_no_repeat_ngram_size,
                              input_ids_seq_length, encoder_input_ids, min_length, max_length, eos_token_id,
                              forced_bos_token_id, forced_eos_token_id, prefix_allowed_tokens_fn, num_beams,
                              num_beam_groups, diversity_penalty, remove_invalid_values,
                              exponential_decay_length_penalty, logits_processor, renormalize_logits):
        processors = LogitsProcessorList()
        repetition_penalty = self._pick(repetition_penalty, "repetition_penalty")
        no_repeat_ngram_size = self._pick(no_repeat_ngram_size, "no_repeat_ngram_size")
        encoder_no_repeat_ngram_size = self._pick(encoder_no_repeat_ngram_size, "encoder_no_repeat_ngram_size")
        min_length = self._pick(min_length, "min_length")
        eos_token_id = self._pick(eos_token_id, "eos_token_id")
        diversity_penalty = self._pick(diversity_penalty, "diversity_penalty")
        forced_bos_token_id = self._pick(forced_bos_token_id, "forced_bos_token_id")
        forced_eos_token_id = self._pick(forced_eos_token_id, "forced_eos_token_id")
        remove_invalid_values = self._pick(remove_invalid_values, "remove_invalid_values")
        exponential_decay_length_penalty = self._pick(exponential_decay_length_penalty, "exponential_decay_length_penalty")
        if diversity_penalty is not None and diversity_penalty > 0.0:
            processors.append(HammingDiversityLogitsProcessor(float(diversity_penalty), num_beams, num_beam_groups))
        if repetition_penalty is not None and repetition_penalty != 1.0:
            processors.append(RepetitionPenaltyLogitsProcessor(float(repetition_penalty)))
        if no_repeat_ngram_size is not None and no_repeat_ngram_size > 0:
            processors.append(NoRepeatNGramLogitsProcessor(no_repeat_ngram_size))
        if encoder_no_repeat_ngram_size is not None and encoder_no_repeat_ngram_size > 0:
            if not self._gcfg("is_encoder_decoder"):
                raise ValueError("It's impossible to use `encoder_no_repeat_ngram_size` with decoder-only architecture")
            processors.append(EncoderNoRepeatNGramLogitsProcessor(encoder_no_repeat_ngram_size, encoder_input_ids))
        if min_length is not None and eos_token_id is not None and min_length > 0:
            processors.append(MinLengthLogitsProcessor(min_length, eos_token_id))
        if prefix_allowed_tokens_fn is not None:
            processors.append(PrefixConstrainedLogitsProcessor(prefix_allowed_tokens_fn, num_beams // num_beam_groups))
        if forced_bos_token_id is not None:
            processors.append(ForcedBOSTokenLogitsProcessor(forced_bos_token_id))
        if forced_eos_token_id is not None:
            processors.append(ForcedEOSTokenLogitsProcessor(max_length, forced_eos_token_id))
        if remove_invalid_values:
            processors.append(InfNanRemoveLogitsProcessor())
        if exponential_decay_length_penalty is not None:
            processors.append(
                ExponentialDecayLengthPenalty(exponential_decay_length_penalty, eos_token_id, input_ids_seq_length)
            )
        processors = self._merge_criteria_processor_list(processors, logits_processor)
        if renormalize_logits:
            processors.append(NormalizationLogitsProcessor())
        return processors

    def _get_stopping_criteria(self, max_length, max_time, stopping_criteria):
        criteria = StoppingCriteriaList()
        if max_length is not None:
            criteria.append(MaxLengthCriteria(max_length=max_length))
        if max_time is not None:
            criteria.append(MaxTimeCriteria(max_time=max_time))
        return self._merge_criteria_processor_list(criteria, stopping_criteria)

    @staticmethod
    def _merge_criteria_processor_list(default_list, custom_list):
        if not custom_list:
            return default_list
        for default in default_list:
            for custom in custom_list:
                if type(custom) is type(default):
                    raise ValueError(
                        f"A custom {type(custom)} was passed to `generate` but one of the same type is already "
                        "created from the arguments; pass different arguments or drop the custom object."
                    )
        default_list.extend(custom_list)
        return default_list

    def compute_transition_beam_scores(self, sequences, scores, beam_indices, eos_token_id=None):
        """Log-prob of every generated token along the returned beams → ``[n_sequences, steps]``.
        ``scores``: per-step ``[batch·beams, vocab]`` tuple from ``beam_search(output_scores=True)``;
        ``beam_indices``: per returned sequence, the beam row it lived in at every step."""
        vocab = scores[0].shape[-1]
        flat = torch.stack(scores).reshape(len(scores), -1).transpose(0, 1)  # [batch·beams·vocab, steps]
        max_len = max(len(b) for b in beam_indices)
        idx = torch.tensor([list(b) + [0] * (max_len - len(b)) for b in beam_indices], device=sequences.device)
        pad = torch.tensor([[False] * len(b) + [True] * (max_len - len(b)) for b in beam_indices], device=sequences.device)
        tokens = sequences[:, sequences.shape[-1] - max_len :]
        tokens = tokens.masked_fill(pad, 0)
        out = flat[:, :max_len].gather(0, idx * vocab + tokens)
        return out.masked_fill(pad, 0)

    def _validate_model_kwargs(self, model_kwargs):
        if self._gcfg("is_encoder_decoder"):
            for key in ("decoder_input_ids",):
                model_kwargs.pop(key, None)
        allowed = set(inspect.signature(self.prepare_inputs_for_generation).parameters)
        if "kwargs" in allowed:
            allowed |= set(inspect.signature(self.forward).parameters)
        unused = [k for k, v in model_kwargs.items() if v is not None and k not in allowed]
        if unused:
            raise ValueError(
                f"The following `model_kwargs` are not used by the model: {unused} (note: typos in the generate "
                "arguments will also show up in this list)"
            )

    # ------------------------------------------------------------------ decoding loops
    def _step_logits(self, outputs):
        logits = outputs["logits"] if "logits" in outputs else outputs["prediction_scores"]
        return logits[:, -1, :].float()

    @staticmethod
    def _sync_tokens(tokens):
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.broadcast(tokens, src=0)
        return tokens

    def _model_inputs(self, input_ids, model_kwargs):
        inputs = self.prepare_inputs_for_generation(input_ids, **model_kwargs)
        return inputs

    # the decode graphs of the running generate() call (decode_graph.DecodeCall), None when its steps run eagerly
    _decode_graphs = None

    def _decode_step(self, input_ids, model_kwargs):
        """One step of the model: replayed from a CUDA graph when ``generate(decode_graphs=True)`` asked for it and the
        step is eligible (:mod:`libai_b200.inference.decode_graph`), else eager."""
        inputs = self._model_inputs(input_ids, model_kwargs)
        if self._decode_graphs is not None:
            return decode_graph.step(self, inputs, self._decode_graphs)
        return self(**inputs)

    @torch.no_grad()
    def greedy_search(self, input_ids, logits_processor=None, stopping_criteria=None, max_length=None,
                      pad_token_id=None, eos_token_id=None, is_encoder_decoder=False, output_scores=False,
                      **model_kwargs):
        logits_processor = logits_processor if logits_processor is not None else LogitsProcessorList()
        stopping_criteria = stopping_criteria if stopping_criteria is not None else StoppingCriteriaList()
        if max_length is not None:
            warnings.warn("`max_length` is deprecated here; use `stopping_criteria=[MaxLengthCriteria(...)]`", UserWarning)
            stopping_criteria = validate_stopping_criteria(stopping_criteria, max_length)
        return self._token_loop(input_ids, lambda s: torch.argmax(s, dim=-1), logits_processor, LogitsProcessorList(),
                                stopping_criteria, pad_token_id, eos_token_id, is_encoder_decoder, output_scores,
                                model_kwargs)

    @torch.no_grad()
    def multinomial_sample(self, input_ids, logits_processor=None, stopping_criteria=None, logits_warper=None,
                           max_length=None, pad_token_id=None, eos_token_id=None, is_encoder_decoder=False,
                           output_scores=False, **model_kwargs):
        logits_processor = logits_processor if logits_processor is not None else LogitsProcessorList()
        stopping_criteria = stopping_criteria if stopping_criteria is not None else StoppingCriteriaList()
        if max_length is not None:
            stopping_criteria = validate_stopping_criteria(stopping_criteria, max_length)
        logits_warper = logits_warper if logits_warper is not None else LogitsProcessorList()
        return self._token_loop(input_ids,
                                lambda s: torch.multinomial(torch.softmax(s, dim=-1), num_samples=1).squeeze(1),
                                logits_processor, logits_warper, stopping_criteria, pad_token_id, eos_token_id,
                                is_encoder_decoder, output_scores, model_kwargs)

    def _token_loop(self, input_ids, pick, logits_processor, logits_warper, stopping_criteria, pad_token_id,
                    eos_token_id, is_encoder_decoder, output_scores, model_kwargs):
        """The loop of ``greedy_search`` and ``multinomial_sample``: one token per step, ``pick`` of the processed and
        warped logits, until every sample has emitted EOS or ``stopping_criteria`` stops."""
        pad_token_id = self._pick(pad_token_id, "pad_token_id")
        eos_token_id = self._pick(eos_token_id, "eos_token_id")
        scores = () if output_scores else None
        unfinished = torch.ones(input_ids.shape[0], dtype=torch.long, device=input_ids.device)
        first = model_kwargs.pop("_first_step", None)   # the outputs of a shared prefill (_shared_prefill)
        while True:
            outputs, first = (self._decode_step(input_ids, model_kwargs) if first is None else first), None
            next_scores = logits_warper(input_ids, logits_processor(input_ids, self._step_logits(outputs)))
            if output_scores:
                scores += (next_scores,)
            next_tokens = pick(next_scores)
            if eos_token_id is not None:
                if pad_token_id is None:
                    raise ValueError("If `eos_token_id` is defined, make sure that `pad_token_id` is defined.")
                next_tokens = next_tokens * unfinished + pad_token_id * (1 - unfinished)
            next_tokens = self._sync_tokens(next_tokens)
            input_ids = torch.cat([input_ids, next_tokens[:, None]], dim=-1)
            model_kwargs = self._update_model_kwargs_for_generation(outputs, model_kwargs, is_encoder_decoder)
            if eos_token_id is not None:
                unfinished = unfinished * (next_tokens != eos_token_id).long()
            if unfinished.max() == 0 or stopping_criteria(input_ids, scores):
                break
        cache = getattr(self, "kv_cache", None)
        if isinstance(cache, PagedKVCache) and cache.fork_n == 1:   # the rows fed: prompt and generated tokens
            cache.insert(input_ids, model_kwargs.get("attention_mask"))
        self._reset_cache()
        return (input_ids, scores) if output_scores else input_ids

    @torch.no_grad()
    def beam_search(self, input_ids, beam_scorer: BeamScorer, logits_processor=None, stopping_criteria=None,
                    max_length=None, pad_token_id=None, eos_token_id=None, is_encoder_decoder=False,
                    output_scores=False, **model_kwargs):
        logits_processor = logits_processor if logits_processor is not None else LogitsProcessorList()
        stopping_criteria = stopping_criteria if stopping_criteria is not None else StoppingCriteriaList()
        if max_length is not None:
            stopping_criteria = validate_stopping_criteria(stopping_criteria, max_length)
        if len(stopping_criteria) == 0:
            warnings.warn("You don't have defined any stopping_criteria, this will likely loop forever", UserWarning)
        pad_token_id = self._pick(pad_token_id, "pad_token_id")
        eos_token_id = self._pick(eos_token_id, "eos_token_id")
        batch_size, num_beams = len(beam_scorer._beam_hyps), beam_scorer.num_beams
        batch_beam_size, cur_len = input_ids.shape
        if num_beams * batch_size != batch_beam_size:
            raise ValueError(f"Batch dimension of `input_ids` should be {num_beams * batch_size}, but is {batch_beam_size}.")
        scores = () if output_scores else None
        beam_indices = tuple(() for _ in range(batch_beam_size)) if output_scores else None
        beam_scores = torch.zeros((batch_size, num_beams), dtype=torch.float32, device=input_ids.device)
        beam_scores[:, 1:] = -1e9  # all beams start identical: only the first one may spawn continuations
        beam_scores = beam_scores.view(-1)
        first = model_kwargs.pop("_first_step", None)   # the outputs of a shared prefill (_shared_prefill)
        while True:
            outputs, first = (self._decode_step(input_ids, model_kwargs) if first is None else first), None
            logprobs = torch.log_softmax(self._step_logits(outputs), dim=-1)
            processed = logits_processor(input_ids, logprobs)
            next_scores = processed + beam_scores[:, None]
            if output_scores:
                scores += (processed,)
            vocab = next_scores.shape[-1]
            next_scores, next_tokens = torch.topk(next_scores.view(batch_size, num_beams * vocab), 2 * num_beams,
                                                  dim=1, largest=True, sorted=True)
            next_indices = torch.div(next_tokens, vocab, rounding_mode="floor")
            next_tokens = next_tokens % vocab
            out = beam_scorer.process(input_ids, next_scores, next_tokens, next_indices, pad_token_id=pad_token_id,
                                      eos_token_id=eos_token_id, beam_indices=beam_indices)
            beam_scores, beam_next, beam_idx = out["next_beam_scores"], out["next_beam_tokens"], out["next_beam_indices"]
            beam_next, beam_idx = self._sync_tokens(beam_next), self._sync_tokens(beam_idx)
            input_ids = torch.cat([input_ids[beam_idx, :], beam_next.unsqueeze(-1)], dim=-1)
            model_kwargs = self._update_model_kwargs_for_generation(outputs, model_kwargs, is_encoder_decoder)
            if model_kwargs.get("past") is not None:
                model_kwargs["past"] = self._reorder_cache(model_kwargs["past"], beam_idx)
                self._apply_reordered_cache(model_kwargs["past"])
            if output_scores:
                beam_indices = tuple(beam_indices[beam_idx[i]] + (int(beam_idx[i]),) for i in range(len(beam_indices)))
            cur_len += 1
            if beam_scorer.is_done or stopping_criteria(input_ids, scores):
                break
        result = beam_scorer.finalize(input_ids, beam_scores, beam_next, beam_idx, pad_token_id=pad_token_id,
                                      eos_token_id=eos_token_id, max_length=stopping_criteria.max_length,
                                      beam_indices=beam_indices)
        self._reset_cache()
        if output_scores:
            return result["sequences"], result["sequence_scores"], scores
        return result["sequences"]

    def _shared_prefill(self, input_ids, n: int, model_kwargs, hit: int = 0):
        """The prefill of the ``b`` prompts once, on a paged cache, which then forks into ``n`` sequences per prompt
        (:meth:`PagedKVCache.fork`).  Other per-sequence inputs given for all ``b * n`` sequences (GLM's positions) are
        taken once per prompt.  ``hit``: the prompts' first ``hit`` pages are mapped from the prefix index already
        (:meth:`PagedKVCache.lookup`), so only the tokens after them are fed; the prompt's full pages are then indexed.
        Returns the expanded ``input_ids`` and ``model_kwargs`` of the decoding loop, whose ``_first_step`` holds the
        prefill's last logits, each prompt's row repeated for its ``n`` sequences."""
        b = input_ids.shape[0]
        once = {k: v[::n] if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == b * n else v
                for k, v in model_kwargs.items()}
        outputs = self._decode_step(input_ids[:, hit * OF.PAGE_ROWS :], once)
        self.kv_cache.insert(input_ids, once.get("attention_mask"))
        self.kv_cache.fork(n)
        key = "logits" if "logits" in outputs else "prediction_scores"
        first = {key: outputs[key][:, -1:].repeat_interleave(n, dim=0)}
        input_ids, model_kwargs = self._expand_inputs_for_generation(input_ids, expand_size=n, **model_kwargs)
        model_kwargs["_first_step"] = first
        return input_ids, model_kwargs

    # a decoder-only model whose cached step takes ``{"input_ids": [b, s], "use_cache": True}`` for any s (positions and
    # padding from its StaticKVCache): it can verify speculative proposals, and serve as a draft
    speculative_decoding = False
    # generate(prefix_cache_tokens=...): a model whose cached rows depend only on the tokens before them
    prefix_caching = True
    # GenerationEngine (continuous batching): a model whose cached step takes positions only from the cache's
    # per-sequence lengths, with continuous_batching_logits and continuous_batching_max_length
    continuous_batching = False

    def _verify_step(self, block):
        """One cached step of the target on ``block`` ``[b, k + 1]`` (a graph of k + 1 tokens when graphs are on)."""
        inputs = {"input_ids": block, "use_cache": True}
        if self._decode_graphs is not None:
            return decode_graph.step(self, inputs, self._decode_graphs, tokens=block.shape[1])
        return self(**inputs)

    @staticmethod
    def _all_logits(outputs):
        return (outputs["logits"] if "logits" in outputs else outputs["prediction_scores"]).contiguous()

    @torch.no_grad()
    def speculative_search(self, input_ids, assistant_model=None, num_assistant_tokens=4, prompt_lookup_num_tokens=None,
                           max_matching_ngram_size=2, stopping_criteria=None, pad_token_id=None, eos_token_id=None,
                           output_scores=False, warp=None, **model_kwargs):
        """Speculative decoding: proposals from ``assistant_model`` (a draft model, ``num_assistant_tokens`` per
        iteration) or from prompt lookup (``prompt_lookup_num_tokens``, :func:`prompt_lookup`), verified in one cached
        step of this model.  Greedy, or speculative sampling with ``warp=(temperature, top_k, top_p)`` (a draft model
        only; below).

        One iteration, x the last emitted token: propose d_1 .. d_k; run the target on ``[x, d_1 .. d_k]``; accept, per
        sample, the longest prefix of the proposals equal to the target's argmaxes; advance the whole batch by the
        minimum n over its unfinished samples and emit the target's tokens t_1 .. t_{n+1} (:func:`OF.spec_accept`, one
        readback per iteration).  The output follows ``greedy_search`` (its shape, EOS padding and stops, one fp32
        score row per emitted token).  Each token equals plain greedy's whenever the verify step's argmax equals the
        single-token step's: the two differ only in rounding (other split ranges in the decode attention, another M
        in the GEMMs), so the output is greedy decoding up to rounding, not bit for bit.

        A sample that emits EOS inside a block, with n past its EOS, is fed the proposals that follow its EOS in that
        block where greedy feeds pad tokens: its cache holds their rows, and its score rows differ from greedy's from
        that position on, in every later iteration too (its tokens are pad either way).  A finished sample's later
        proposals are pad tokens.

        After every iteration each cache holds the rows of the sequence minus its last token, as greedy leaves them
        (but for the rows after a finished sample's EOS, above):
        the target drops the rows past the accepted tokens (``StaticKVCache.rollback``); the draft, which only takes
        single-token steps, rolls back too, or, when all k were accepted, feeds d_k at the start of the next
        iteration.  Both caches hold ``max_length + k`` rows (``generate`` sizes them).  Near a model's maximum
        positions k shrinks so that no step writes past them; those steps run eagerly under decode graphs.

        Speculative sampling (``warp`` given; Leviathan et al. 2023, Chen et al. 2023): p and q are the target's and
        the draft's distributions under one warp rule (temperature, top-k, top-p: :func:`OF.spec_warp_ref`).  After
        each of its k single-token steps the draft samples d_{j+1} ~ q_j on the device (:func:`OF.spec_sample`, uniforms
        ``[b, k]`` from ``torch.rand``) and keeps its logits row; after the verify step :func:`OF.spec_accept_sample`
        accepts d_{j+1} with probability min(1, p_j/q_j) and replaces the first rejected one by a draw from
        norm(max(0, p_j − q_j)), or draws a bonus token from p_k when all are accepted (uniforms ``[b, k + 1, 2]``).
        The batch advances by the same n and the caches roll back as above.  Every emitted token is distributed as p
        given its prefix, whatever the draft is.  Each iteration draws a fixed number of uniforms from the default
        generator, so ``torch.manual_seed`` reproduces a call, eagerly or under decode graphs.  ``output_scores``
        holds the target's warped logits (z on the kept set, −inf elsewhere), as ``multinomial_sample`` reports them."""
        stopping_criteria = stopping_criteria if stopping_criteria is not None else StoppingCriteriaList()
        draft = assistant_model
        k = num_assistant_tokens if draft is not None else prompt_lookup_num_tokens
        max_length = stopping_criteria.max_length
        b, dev = input_ids.shape[0], input_ids.device
        scores = () if output_scores else None
        sample = warp is not None
        if sample and draft is None:
            raise ValueError("do_sample: speculative sampling needs an assistant_model (prompt lookup has no proposal "
                             "distribution)")

        outputs = self._decode_step(input_ids, model_kwargs)
        cache = self.kv_cache
        if cache.dense_mask:
            raise ValueError("attention_mask: speculative decoding needs padding that the cache's kv_start holds "
                             "(left padding); this prompt needs a dense mask")
        rows = self._all_logits(outputs)[:, -1:].contiguous()
        # per model: the rows its cache holds besides the sequence's (ChatGLM's P-tuning prefix), and the rows an
        # iteration's steps write besides the k proposals (the verify step's x)
        models = [(self, cache.length - input_ids.shape[1], 1)]
        draft_kwargs = {"past": None, "use_cache": True}
        if draft is not None:
            mask = model_kwargs.get("attention_mask")
            draft_out = draft._decode_step(input_ids, {"use_cache": True, **({} if mask is None else
                                                                            {"attention_mask": mask})})
            if draft._all_logits(draft_out).shape[-1] != rows.shape[-1]:
                raise ValueError(f"assistant_model: its logits are {draft._all_logits(draft_out).shape[-1]} wide, the "
                                 f"target's {rows.shape[-1]}")
            if draft.kv_cache.dense_mask:
                raise ValueError("attention_mask: the assistant's cache needs a dense mask for this prompt")
            draft_kwargs["past"] = draft.kv_cache
            models.append((draft, draft.kv_cache.length - input_ids.shape[1], 0))
            if sample:   # the draft's logits rows of an iteration, from which the acceptance recomputes q
                qbuf = torch.empty(b, k, rows.shape[-1], dtype=draft._all_logits(draft_out).dtype, device=dev)
        history = staging = None
        if draft is None:
            history = input_ids.tolist()
            if dev.type == "cuda":   # prompt-lookup proposals reach the device by an asynchronous copy from pinned memory
                staging = torch.empty(b * k, dtype=input_ids.dtype, pin_memory=True)
        proposals = input_ids.new_empty(b, 0)
        unfinished = torch.ones(b, dtype=torch.long, device=dev)
        host_unfinished = [1] * b
        while True:
            R = rows.shape[1]
            if sample:
                u = torch.rand(b, R, 2, device=dev)
                warped = torch.empty(rows.shape, dtype=torch.float32, device=dev) if output_scores else None
                res = OF.spec_accept_sample(rows, qbuf, proposals, u, unfinished, *warp, eos_token_id, pad_token_id,
                                            warped)
            else:
                res = OF.spec_accept(rows, proposals, unfinished, eos_token_id, pad_token_id)
            host = res.tolist()   # the iteration's one readback
            n = host[0][2 * R + 1]
            count = n + 1
            if max_length is not None:
                count = min(count, max(max_length - input_ids.shape[1], 1))   # greedy emits one token at least
            if eos_token_id is not None:   # greedy stops at the first position where every sample is finished
                live = list(host_unfinished)
                for j in range(count):
                    live = [u and int(host[i][R + j] != eos_token_id) for i, u in enumerate(live)]
                    if not any(live):
                        count = j + 1
                        break
            input_ids = torch.cat([input_ids, res[:, R : R + count]], dim=-1)
            if output_scores:
                scores += tuple(warped[:, j] if sample else rows[:, j].float() for j in range(count))
            if history is not None:
                for i in range(b):
                    history[i].extend(host[i][R : R + count])
            host_unfinished = [row[2 * R + 2] for row in host]
            if not any(host_unfinished) or count < n + 1 or stopping_criteria(input_ids, scores):
                break

            # both caches back to the invariant: the rows of the sequence minus its last token; then k, so that no
            # step writes past a model's maximum positions
            L = input_ids.shape[1]
            kk = k
            for m, m_extra, more in models:
                c, held = m.kv_cache, L - 1 + m_extra
                if c.length < held:   # every proposal was accepted: the draft lacks the row of d_k
                    draft._decode_step(input_ids[:, L - 2 : L - 1], draft_kwargs)
                else:
                    c.rollback(c.length - held)
                    m.past_length = c.length
                if m.max_cache_positions is not None:
                    kk = min(kk, m.max_cache_positions - c.length - more)
            kk = max(kk, 0)

            x = input_ids[:, -1:]
            if draft is not None:
                if sample:
                    ud = torch.rand(b, kk, device=dev)
                proposals, tok = input_ids.new_empty(b, kk), x
                for j in range(kk):
                    step = self._all_logits(draft._decode_step(tok, draft_kwargs))[:, -1]
                    if sample:
                        OF.spec_sample(step, qbuf, j, ud, proposals, *warp)
                    else:
                        proposals[:, j] = step.argmax(dim=-1)
                    tok = proposals[:, j : j + 1].contiguous()
            else:
                proposals = torch.tensor([prompt_lookup(h, kk, max_matching_ngram_size) for h in history],
                                         dtype=input_ids.dtype).view(b, kk)
                if staging is not None:
                    # the previous iteration's copy out of the buffer ended before its readback returned
                    proposals = staging[: b * kk].view(b, kk).copy_(proposals)
                proposals = proposals.to(dev, non_blocking=True)
            if eos_token_id is not None:   # a finished sample is fed pad tokens, as greedy feeds it
                proposals = proposals.masked_fill(unfinished[:, None] == 0, pad_token_id)
            rows = self._all_logits(self._verify_step(torch.cat([x, proposals], dim=1)))
        self._reset_cache()
        if draft is not None:
            draft._reset_cache()
        return (input_ids, scores) if output_scores else input_ids

    def _speculative_args(self, draft, num_assistant_tokens, prompt_lookup_num_tokens, max_matching_ngram_size,
                          do_sample, num_beams, num_return_sequences, processors, custom_criteria, is_enc_dec,
                          max_length, model_kwargs, temperature=None, top_k=None, top_p=None, typical_p=None):
        """Check a speculative ``generate()`` call; returns ``(k, max_matching_ngram_size, warp)``, warp the
        ``(temperature, top_k, top_p)`` of speculative sampling (None when greedy)."""
        if draft is not None and prompt_lookup_num_tokens is not None:
            raise ValueError("assistant_model and prompt_lookup_num_tokens: give one proposer, not both")
        name = "assistant_model" if draft is not None else "prompt_lookup_num_tokens"
        k = (4 if num_assistant_tokens is None else num_assistant_tokens) if draft is not None \
            else prompt_lookup_num_tokens
        arg = "num_assistant_tokens" if draft is not None else "prompt_lookup_num_tokens"
        if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= MAX_SPECULATIVE_TOKENS:
            raise ValueError(f"{arg} must be an int in [1, {MAX_SPECULATIVE_TOKENS}], got {k!r}")
        ngram = 2 if max_matching_ngram_size is None else max_matching_ngram_size
        if draft is None and (isinstance(ngram, bool) or not isinstance(ngram, int) or ngram < 1):
            raise ValueError(f"max_matching_ngram_size must be a positive int, got {ngram!r}")
        if do_sample and draft is None:
            raise ValueError(f"{name}: do_sample=True needs an assistant_model; prompt lookup has no proposal "
                             "distribution to sample from")
        if num_beams != 1:
            raise ValueError(f"{name}: speculative decoding does not search beams; num_beams={num_beams} is not "
                             "supported")
        if num_return_sequences != 1 and not do_sample:
            raise ValueError(f"{name}: num_return_sequences={num_return_sequences} needs do_sample=True")
        warp = None
        if do_sample:
            # the warpers multinomial_sample would apply, validated by their classes; the kernels apply the same rule
            self._get_logits_warper(top_k, top_p, typical_p, temperature, num_beams)
            typical_p = self._pick(typical_p, "typical_p")
            if typical_p is not None and typical_p < 1.0:
                raise ValueError(f"{name}: speculative sampling applies temperature, top_k and top_p; "
                                 f"typical_p={typical_p} is not supported")
            temperature, top_k, top_p = (self._pick(v, key) for v, key in ((temperature, "temperature"),
                                                                            (top_k, "top_k"), (top_p, "top_p")))
            top_p = 1.0 if top_p is None or top_p >= 1.0 else float(top_p)
            if not top_p > 0:
                raise ValueError(f"{name}: speculative sampling needs top_p > 0, got {top_p}")
            warp = (1.0 if temperature is None else float(temperature), 0 if top_k is None else int(top_k), top_p)
        if processors:
            names = sorted({_PROCESSOR_ARGS.get(type(p), "logits_processor") for p in processors})
            raise ValueError(f"{name}: speculative decoding applies no logits processor; drop {', '.join(names)}")
        if custom_criteria:
            raise ValueError(f"{name}: custom stopping_criteria are not supported (max_length and max_time are)")
        if not model_kwargs.get("use_cache"):
            raise ValueError(f"{name}: speculative decoding runs on the KV cache; use_cache=False is not supported")
        if max_length is None:
            raise ValueError(f"{name}: speculative decoding sizes both caches from max_length; give max_length or "
                             "max_new_tokens")
        topo = dutil.get_dist_util()
        if topo.tensor_parallel_size > 1 or topo.pipeline_parallel_size > 1:
            raise ValueError(f"{name}: tensor- or pipeline-parallel inference is not supported")
        for role, m in (("the model", self), ("assistant_model", draft)):
            if m is None:
                continue
            cls = type(m).__name__
            if not (isinstance(m, KVCacheOwner) and isinstance(m, Generator)) or not m.speculative_decoding or \
                    bool(m._gcfg("is_encoder_decoder")) or (m is self and is_enc_dec):
                raise ValueError(f"{name}: {role} ({cls}) is not a decoder-only model that speculative decoding "
                                 "supports (encoder-decoder and GLM models are not)")
        if draft is not None:
            if draft is self:
                raise ValueError("assistant_model must be another model than the one generating: each owns one cache")
            if draft._device() != self._device():
                raise ValueError(f"assistant_model is on {draft._device()}, the model on {self._device()}")
        return k, ngram, warp

    # ------------------------------------------------------------------ entry point
    @torch.no_grad()
    def generate(self, inputs=None, max_length=None, min_length=None, do_sample=None, early_stopping=None,
                 num_beams=None, temperature=None, top_k=None, top_p=None, typical_p=None, repetition_penalty=None,
                 force_words_ids=None, bos_token_id=None, pad_token_id=None, eos_token_id=None, length_penalty=None,
                 no_repeat_ngram_size=None, encoder_no_repeat_ngram_size=None, num_return_sequences=None,
                 max_time=None, max_new_tokens=None, decoder_start_token_id=None, use_cache=None,
                 num_beam_groups=None, diversity_penalty=None, prefix_allowed_tokens_fn=None, logits_processor=None,
                 renormalize_logits=None, stopping_criteria=None, constraints=None, output_scores=None,
                 forced_bos_token_id=None, forced_eos_token_id=None, remove_invalid_values=None,
                 exponential_decay_length_penalty=None, kv_cache_dtype=None, decode_graphs=None, assistant_model=None,
                 num_assistant_tokens=None, prompt_lookup_num_tokens=None, max_matching_ngram_size=None,
                 paged_kv_cache=None, prefix_cache_tokens=None, **model_kwargs):
        """``kv_cache_dtype`` (default: the model cfg's ``kv_cache_dtype``): ``"fp8"`` or ``torch.float8_e4m3fn`` holds
        the preallocated KV cache as E4M3 rows with per-row scales
        (:class:`~libai_b200.inference.kv_cache.StaticKVCache`) for this call: about half the memory, and of the bytes
        each decoding step reads, for 8-bit keys and values.
        None keeps the weights' dtype.  A model that does not decode on a ``StaticKVCache`` raises ``ValueError``.

        ``decode_graphs`` (default: the model cfg's ``decode_graphs``, else False): True replays the cached decode steps
        from a CUDA graph, one graph launch per step (:mod:`libai_b200.inference.decode_graph`), with the tokens of
        eager decoding.  The first decode step of a new batch or cache runs eagerly and the next is captured; the
        graph holds a private memory pool while the cache lives, and Python hooks on modules do not run in a replayed
        step.  Steps the graph cannot reproduce run eagerly (logged once per reason).  A model that does not decode on
        a ``StaticKVCache`` raises ``ValueError``.

        Speculative decoding (:meth:`speculative_search`): ``assistant_model`` (a second decoder-only
        model on the same device, with the same logits width; ``num_assistant_tokens`` proposals per iteration, 1 to
        15, default 4) or ``prompt_lookup_num_tokens`` (1 to 15 proposals from the sequence itself, matching n-grams of
        up to ``max_matching_ngram_size`` tokens, default 2), not both.  ``kv_cache_dtype`` applies to this model, the
        assistant's cfg sets its own; ``decode_graphs`` applies to both.  Greedy, or with ``do_sample=True`` and an
        ``assistant_model``, speculative sampling: ``temperature``, ``top_k`` and ``top_p`` (``generate()``'s defaults,
        so top-k 50) warp both models' logits, and the output follows the target's warped distribution exactly;
        ``num_return_sequences`` expands the inputs as ``multinomial_sample`` does.  Beams, ``typical_p < 1``,
        ``do_sample`` with prompt lookup, ``num_return_sequences > 1`` without sampling, logits processors (including
        ``renormalize_logits``), custom stopping criteria, encoder-decoder and GLM models, tensor or pipeline
        parallelism and a prompt whose padding needs a dense mask raise ``ValueError``.

        ``paged_kv_cache`` (default: the model cfg's ``paged_kv_cache``, else False): True holds the cache in 64-row
        pages (:class:`~libai_b200.inference.kv_cache.PagedKVCache`), with the tokens of the contiguous cache.  Beam
        search, and sampling with ``num_return_sequences > 1``, then prefill each prompt once and fork its cache into
        the beams or samples, which share the prompt's pages; a beam reorder rewrites block tables instead of copying
        the cache.  Greedy search and single-sequence sampling run on pages without a fork.  Encoder-decoder models
        (T5/mT5) and models without a preallocated cache, tensor or pipeline parallelism, and speculative decoding
        raise ``ValueError``.

        ``prefix_cache_tokens`` (default: the model cfg's ``prefix_cache_tokens``, else 0 = off): N > 0 keeps up to N
        tokens (rounded up to 64-row pages) of K/V pages across calls, on a paged cache (it implies
        ``paged_kv_cache=True``; an explicit ``paged_kv_cache=False`` raises ``ValueError``).  A call whose prompts all
        start with cached pages maps them and prefills only the rest (at least one token); ``kv_cache.reused_rows``
        counts the rows taken.  A page is keyed by the tokens and padding mask of its rows and of every row before it,
        so a left-padded prompt matches prompts with the same padding.  After the prefill the prompt's full pages are
        cached; after a greedy or single-sample call also those of its generated tokens, so the next chat turn reuses its
        previous answer.  The pool and its index are kept while later calls fit the pool (batch, sequences per prompt,
        length and cache format), and are cleared when a parameter or the KV dtype changes, or by
        ``clear_prefix_cache()``.  The first tokens' logits are not bitwise those of a full prefill (the GEMMs see
        another number of rows).  Prompts whose padding needs a dense mask, and caches with rows before the prompt
        (ChatGLM's P-tuning), are neither looked up nor cached.  The cases ``paged_kv_cache`` refuses, and GLM (whose
        prefix-LM prompt attends bidirectionally), raise ``ValueError``."""
        kv_cache_dtype = _kv_cache_dtype(self._pick(kv_cache_dtype, "kv_cache_dtype"))
        prefix_tokens = _prefix_cache_tokens(self._pick(prefix_cache_tokens, "prefix_cache_tokens"))
        if prefix_tokens > 0 and paged_kv_cache is False:
            raise ValueError("prefix_cache_tokens > 0 holds the cache in pages: it cannot run with paged_kv_cache=False")
        paged = prefix_tokens > 0 or _paged_kv_cache(self._pick(paged_kv_cache, "paged_kv_cache"))
        if paged:
            what = "prefix_cache_tokens > 0" if prefix_tokens > 0 else "paged_kv_cache=True"
            if not isinstance(self, KVCacheOwner) or self._gcfg("is_encoder_decoder"):
                raise ValueError(f"{what}: {type(self).__name__} is not a decoder-only model with a "
                                 "preallocated KV cache")
            topo = dutil.get_dist_util()
            if topo.tensor_parallel_size > 1 or topo.pipeline_parallel_size > 1:
                raise ValueError(f"{what}: tensor- and pipeline-parallel inference keep contiguous caches")
            if assistant_model is not None or prompt_lookup_num_tokens is not None:
                raise ValueError(f"{what}: speculative decoding (assistant_model, prompt_lookup_num_tokens) "
                                 "runs on contiguous caches")
            if prefix_tokens > 0 and not self.prefix_caching:
                raise ValueError(f"prefix_cache_tokens > 0: {type(self).__name__}'s cached rows depend on later "
                                 "tokens (a bidirectional prompt), so they cannot be reused")
        if kv_cache_dtype is not None and not isinstance(self, KVCacheOwner):
            raise ValueError(f"kv_cache_dtype={kv_cache_dtype}: {type(self).__name__} does not decode on a "
                             "StaticKVCache")
        decode_graphs = _decode_graphs(self._pick(decode_graphs, "decode_graphs"))
        if decode_graphs and not isinstance(self, KVCacheOwner):
            raise ValueError(f"decode_graphs=True: {type(self).__name__} does not decode on a StaticKVCache")
        self._validate_model_kwargs(model_kwargs.copy())
        logits_processor = logits_processor if logits_processor is not None else LogitsProcessorList()
        stopping_criteria = stopping_criteria if stopping_criteria is not None else StoppingCriteriaList()
        is_enc_dec = bool(self._gcfg("is_encoder_decoder"))
        bos_token_id = self._pick(bos_token_id, "bos_token_id")
        num_beams = self._pick(num_beams, "num_beams")
        length_penalty = self._pick(length_penalty, "length_penalty")
        early_stopping = self._pick(early_stopping, "early_stopping")
        num_beam_groups = self._pick(num_beam_groups, "num_beam_groups")
        do_sample = self._pick(do_sample, "do_sample")
        num_return_sequences = self._pick(num_return_sequences, "num_return_sequences")
        pad_token_id = self._pick(pad_token_id, "pad_token_id")
        eos_token_id = self._pick(eos_token_id, "eos_token_id")
        output_scores = self._pick(output_scores, "output_scores")
        if pad_token_id is None and eos_token_id is not None:
            logger.warning(f"Setting `pad_token_id` to `eos_token_id`:{eos_token_id} for open-end generation.")
            pad_token_id = eos_token_id

        inputs_tensor, model_input_name, model_kwargs = self._prepare_model_inputs(inputs, bos_token_id, model_kwargs)
        inputs_tensor = inputs_tensor.to(self._device())
        batch_size = inputs_tensor.shape[0]
        model_kwargs["use_cache"] = self._pick(use_cache, "use_cache")
        self._reset_cache()

        mask_name = "encoder_attn_mask" if is_enc_dec else "attention_mask"
        accepts_mask = mask_name in inspect.signature(self.forward).parameters
        if model_kwargs.get(mask_name) is None and accepts_mask and "encoder_outputs" not in model_kwargs:
            model_kwargs[mask_name] = self._prepare_attention_mask_for_generation(inputs_tensor, pad_token_id, eos_token_id)
        elif model_kwargs.get(mask_name) is not None:
            model_kwargs[mask_name] = model_kwargs[mask_name].to(self._device())

        if is_enc_dec:
            model_kwargs = self._prepare_encoder_decoder_kwargs_for_generation(inputs_tensor, model_kwargs, model_input_name)
            input_ids = self._prepare_decoder_input_ids_for_generation(
                batch_size, decoder_start_token_id=decoder_start_token_id, bos_token_id=bos_token_id,
                model_kwargs=model_kwargs,
            )
        else:
            input_ids = inputs_tensor

        input_ids_seq_length = input_ids.shape[-1]
        if max_length is None and max_new_tokens is None:
            max_length = self._gcfg("max_length")
        elif max_length is None and max_new_tokens is not None:
            max_length = max_new_tokens + input_ids_seq_length
        elif max_length is not None and max_new_tokens is not None:
            raise ValueError("Both `max_new_tokens` and `max_length` have been set but they serve the same purpose.")
        min_length = self._pick(min_length, "min_length")
        if min_length is not None and min_length > max_length:
            raise ValueError(f"Unfeasible length constraints: min_length ({min_length}) > max_length ({max_length})")
        if input_ids_seq_length >= max_length:
            logger.warning(
                f"Input length is {input_ids_seq_length}, but `max_length` is set to {max_length}. "
                "This can lead to unexpected behavior. You should consider increasing `max_new_tokens`."
            )

        if constraints is not None or force_words_ids is not None:
            raise NotImplementedError("constrained beam search is not supported (neither is it in the reference)")
        is_greedy = num_beams == 1 and num_beam_groups == 1 and not do_sample
        is_sample = num_beams == 1 and num_beam_groups == 1 and do_sample
        is_beam = num_beams > 1 and num_beam_groups == 1 and not do_sample
        if num_beam_groups > num_beams:
            raise ValueError("`num_beam_groups` has to be smaller or equal to `num_beams`")
        if num_beam_groups > 1:
            raise NotImplementedError("group beam search is not supported (neither is it in the reference)")

        logits_processor = self._get_logits_processor(
            repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size,
            encoder_no_repeat_ngram_size=encoder_no_repeat_ngram_size, input_ids_seq_length=input_ids_seq_length,
            encoder_input_ids=inputs_tensor, min_length=min_length, max_length=max_length, eos_token_id=eos_token_id,
            forced_bos_token_id=forced_bos_token_id, forced_eos_token_id=forced_eos_token_id,
            prefix_allowed_tokens_fn=prefix_allowed_tokens_fn, num_beams=num_beams, num_beam_groups=num_beam_groups,
            diversity_penalty=diversity_penalty, remove_invalid_values=remove_invalid_values,
            exponential_decay_length_penalty=exponential_decay_length_penalty, logits_processor=logits_processor,
            renormalize_logits=renormalize_logits,
        )
        custom_criteria = bool(stopping_criteria)
        stopping_criteria = self._get_stopping_criteria(max_length, max_time, stopping_criteria)
        draft = assistant_model
        speculative = draft is not None or prompt_lookup_num_tokens is not None
        spec_k, spec_warp = 0, None
        if speculative:
            spec_k, max_matching_ngram_size, spec_warp = self._speculative_args(
                draft, num_assistant_tokens, prompt_lookup_num_tokens, max_matching_ngram_size, do_sample, num_beams,
                num_return_sequences, logits_processor, custom_criteria, is_enc_dec, stopping_criteria.max_length,
                model_kwargs, temperature=temperature, top_k=top_k, top_p=top_p, typical_p=typical_p)
        # sequences per prompt: a paged cache forks into them after one prefill per prompt
        fork = num_beams if is_beam else num_return_sequences if is_sample else 1
        with contextlib.ExitStack() as call:
            call.enter_context(_call_state(self, kv_cache_dtype, decode_graphs,
                                           (fork, input_ids_seq_length, prefix_tokens) if paged else None))
            models = [self]
            if draft is not None:   # the assistant's cfg sets its cache format
                call.enter_context(_call_state(draft, _kv_cache_dtype(draft._gcfg("kv_cache_dtype")), decode_graphs))
                models.insert(0, draft)
            # models with a preallocated cache size it once for every sequence the search runs; a verify step appends
            # k + 1 rows and keeps n + 1 of them: room for k more than the output
            rows = batch_size * (1 if paged else fork)
            for m in models:
                allocate = getattr(m, "allocate_kv_cache", None)
                if allocate is not None and model_kwargs.get("use_cache") and stopping_criteria.max_length is not None:
                    if allocate(rows, stopping_criteria.max_length + spec_k) is None and kv_cache_dtype is not None:
                        raise ValueError(f"kv_cache_dtype={kv_cache_dtype}: {type(m).__name__} keeps a tuple cache "
                                         "here (pipeline-parallel inference), not a StaticKVCache")
            if speculative:
                if is_sample:   # as multinomial_sample expands them
                    input_ids, model_kwargs = self._expand_inputs_for_generation(
                        input_ids, expand_size=num_return_sequences, is_encoder_decoder=is_enc_dec, **model_kwargs)
                return self.speculative_search(
                    input_ids, assistant_model=draft, num_assistant_tokens=spec_k,
                    prompt_lookup_num_tokens=spec_k if draft is None else None,
                    max_matching_ngram_size=max_matching_ngram_size, stopping_criteria=stopping_criteria,
                    pad_token_id=pad_token_id, eos_token_id=eos_token_id, output_scores=output_scores, warp=spec_warp,
                    **model_kwargs)
            # the prefix index: map the prompts' cached pages, then prefill the rest once (_shared_prefill)
            hit, prefix = 0, prefix_tokens > 0 and model_kwargs.get("use_cache") and isinstance(self.kv_cache,
                                                                                                PagedKVCache)
            if prefix:
                cache = self.kv_cache
                if self.cache_rows_before_prompt:
                    cache.prefix_ok = False
                else:
                    hit = cache.lookup(input_ids, model_kwargs.get("attention_mask"))
            if is_greedy:
                if num_return_sequences > 1:
                    raise ValueError(f"num_return_sequences has to be 1, but is {num_return_sequences} when doing greedy search.")
                if prefix:
                    input_ids, model_kwargs = self._shared_prefill(input_ids, 1, model_kwargs, hit)
                return self.greedy_search(input_ids, logits_processor=logits_processor,
                                          stopping_criteria=stopping_criteria, pad_token_id=pad_token_id,
                                          eos_token_id=eos_token_id, is_encoder_decoder=is_enc_dec,
                                          output_scores=output_scores, **model_kwargs)
            shared = (fork > 1 or prefix) and model_kwargs.get("use_cache") and isinstance(self.kv_cache, PagedKVCache)
            if is_sample:
                warper = self._get_logits_warper(top_k, top_p, typical_p, temperature, num_beams, renormalize_logits)
                if shared:
                    input_ids, model_kwargs = self._shared_prefill(input_ids, fork, model_kwargs, hit)
                else:
                    input_ids, model_kwargs = self._expand_inputs_for_generation(
                        input_ids, expand_size=num_return_sequences, is_encoder_decoder=is_enc_dec, **model_kwargs)
                return self.multinomial_sample(input_ids, logits_processor=logits_processor, logits_warper=warper,
                                               stopping_criteria=stopping_criteria, pad_token_id=pad_token_id,
                                               eos_token_id=eos_token_id, is_encoder_decoder=is_enc_dec,
                                               output_scores=output_scores, **model_kwargs)
            if is_beam:
                if num_return_sequences > num_beams:
                    raise ValueError("`num_return_sequences` has to be smaller or equal to `num_beams`.")
                if stopping_criteria.max_length is None:
                    raise ValueError("`max_length` needs to be a stopping_criteria for now.")
                scorer = BeamSearchScorer(batch_size=batch_size, num_beams=num_beams, length_penalty=length_penalty,
                                          do_early_stopping=early_stopping, num_beam_hyps_to_keep=num_return_sequences)
                if shared:
                    input_ids, model_kwargs = self._shared_prefill(input_ids, fork, model_kwargs, hit)
                else:
                    input_ids, model_kwargs = self._expand_inputs_for_generation(
                        input_ids, expand_size=num_beams, is_encoder_decoder=is_enc_dec, **model_kwargs)
                return self.beam_search(input_ids, scorer, logits_processor=logits_processor,
                                        stopping_criteria=stopping_criteria, pad_token_id=pad_token_id,
                                        eos_token_id=eos_token_id, is_encoder_decoder=is_enc_dec,
                                        output_scores=output_scores, **model_kwargs)
            raise NotImplementedError("beam sampling is not supported (neither is it in the reference)")
