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

import inspect
import logging
import warnings
from typing import Callable, Dict, Iterable, List, Optional, Tuple, Union

import torch

from libai_b200.utils import distributed as dutil
import torch.distributed as dist

from ..kv_cache import StaticKVCache
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
)


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

    @torch.no_grad()
    def greedy_search(self, input_ids, logits_processor=None, stopping_criteria=None, max_length=None,
                      pad_token_id=None, eos_token_id=None, is_encoder_decoder=False, output_scores=False,
                      **model_kwargs):
        logits_processor = logits_processor if logits_processor is not None else LogitsProcessorList()
        stopping_criteria = stopping_criteria if stopping_criteria is not None else StoppingCriteriaList()
        if max_length is not None:
            warnings.warn("`max_length` is deprecated here; use `stopping_criteria=[MaxLengthCriteria(...)]`", UserWarning)
            stopping_criteria = validate_stopping_criteria(stopping_criteria, max_length)
        pad_token_id = self._pick(pad_token_id, "pad_token_id")
        eos_token_id = self._pick(eos_token_id, "eos_token_id")
        scores = () if output_scores else None
        unfinished = torch.ones(input_ids.shape[0], dtype=torch.long, device=input_ids.device)
        while True:
            outputs = self(**self._model_inputs(input_ids, model_kwargs))
            next_scores = logits_processor(input_ids, self._step_logits(outputs))
            if output_scores:
                scores += (next_scores,)
            next_tokens = torch.argmax(next_scores, dim=-1)
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
        self._reset_cache()
        return (input_ids, scores) if output_scores else input_ids

    @torch.no_grad()
    def multinomial_sample(self, input_ids, logits_processor=None, stopping_criteria=None, logits_warper=None,
                           max_length=None, pad_token_id=None, eos_token_id=None, is_encoder_decoder=False,
                           output_scores=False, **model_kwargs):
        logits_processor = logits_processor if logits_processor is not None else LogitsProcessorList()
        stopping_criteria = stopping_criteria if stopping_criteria is not None else StoppingCriteriaList()
        if max_length is not None:
            stopping_criteria = validate_stopping_criteria(stopping_criteria, max_length)
        logits_warper = logits_warper if logits_warper is not None else LogitsProcessorList()
        pad_token_id = self._pick(pad_token_id, "pad_token_id")
        eos_token_id = self._pick(eos_token_id, "eos_token_id")
        scores = () if output_scores else None
        unfinished = torch.ones(input_ids.shape[0], dtype=torch.long, device=input_ids.device)
        while True:
            outputs = self(**self._model_inputs(input_ids, model_kwargs))
            next_scores = logits_warper(input_ids, logits_processor(input_ids, self._step_logits(outputs)))
            if output_scores:
                scores += (next_scores,)
            probs = torch.softmax(next_scores, dim=-1)
            next_tokens = torch.multinomial(probs, num_samples=1).squeeze(1)
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
        while True:
            outputs = self(**self._model_inputs(input_ids, model_kwargs))
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
                 exponential_decay_length_penalty=None, **model_kwargs):
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
        stopping_criteria = self._get_stopping_criteria(max_length, max_time, stopping_criteria)
        # models with a preallocated cache size it once for every sequence the search runs
        allocate = getattr(self, "allocate_kv_cache", None)
        if allocate is not None and model_kwargs.get("use_cache") and stopping_criteria.max_length is not None:
            rows = batch_size * (num_beams if is_beam else num_return_sequences if is_sample else 1)
            allocate(rows, stopping_criteria.max_length)

        was_training = self.training
        self.eval()
        try:
            if is_greedy:
                if num_return_sequences > 1:
                    raise ValueError(f"num_return_sequences has to be 1, but is {num_return_sequences} when doing greedy search.")
                return self.greedy_search(input_ids, logits_processor=logits_processor,
                                          stopping_criteria=stopping_criteria, pad_token_id=pad_token_id,
                                          eos_token_id=eos_token_id, is_encoder_decoder=is_enc_dec,
                                          output_scores=output_scores, **model_kwargs)
            if is_sample:
                warper = self._get_logits_warper(top_k, top_p, typical_p, temperature, num_beams, renormalize_logits)
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
                input_ids, model_kwargs = self._expand_inputs_for_generation(
                    input_ids, expand_size=num_beams, is_encoder_decoder=is_enc_dec, **model_kwargs)
                return self.beam_search(input_ids, scorer, logits_processor=logits_processor,
                                        stopping_criteria=stopping_criteria, pad_token_id=pad_token_id,
                                        eos_token_id=eos_token_id, is_encoder_decoder=is_enc_dec,
                                        output_scores=output_scores, **model_kwargs)
            raise NotImplementedError("beam sampling is not supported (neither is it in the reference)")
        finally:
            self.train(was_training)
