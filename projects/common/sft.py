"""Shared pieces of the instruction-tuning (SFT) projects (Llama, Aquila, Baichuan, Qwen, ChatGLM):

* ``SFTDataset`` — ``torch.save``-d list of ``{"input_ids", "labels"}`` produced by ``prepare_sft_corpus``
  (reference projects/Llama/dataset.py:8-22 and its copies in the sibling projects);
* ``PackedSFTDataset`` — the same corpus packed several samples to a row, with per-document ``position_ids`` (the
  Llama family attends and rotates per document, so no compute goes to padding between samples);
* ``generate_prompt`` / ``prepare_sample`` / ``prepare_sft_corpus`` — Alpaca-style prompt construction, tokenisation,
  prompt masking (label −1 = ignored) and fixed-length padding (reference projects/Llama/utils/prepare_alpaca.py);
* ``SentencePieceTokenizer`` — the minimal sentencepiece wrapper those projects use (reference
  projects/Llama/tokenizer.py:16-110), returning ``torch`` tensors.
"""
from __future__ import annotations

import json
import os
import random
from typing import List, Optional

import torch
from torch.utils.data import Dataset

from libai_b200.data.structures import DistTensorData, Instance

IGNORE_INDEX = -1


class SFTDataset(Dataset):
    def __init__(self, path, tokenizer=None):
        self.data = torch.load(path, weights_only=False) if isinstance(path, (str, os.PathLike)) else list(path)
        self.tokenizer = tokenizer

    def __len__(self):
        return len(self.data)

    def __getitem__(self, index):
        item = self.data[index]
        return Instance(
            input_ids=DistTensorData(torch.as_tensor(item["input_ids"], dtype=torch.long)),
            labels=DistTensorData(torch.as_tensor(item["labels"], dtype=torch.long), placement_idx=-1),
        )


def sample_length(labels) -> int:
    """Tokens of a prepared sample that matter for training: up to the input that predicts its last trainable label
    (label > 0; ``SFTLoss`` ignores 0 and ``IGNORE_INDEX``), plus the token that label names, i.e. the last trainable
    label's index + 2.  0 for a sample without a trainable label."""
    idx = torch.nonzero(torch.as_tensor(labels) > 0).flatten()
    return int(idx[-1]) + 2 if idx.numel() else 0


def pack_samples(lengths, max_length: int) -> List[List[int]]:
    """Sample indices per row: samples are taken in order and a row is closed when the next one does not fit, so the
    packing is deterministic, keeps the corpus order and never splits a sample.  Samples of length 0 are dropped."""
    rows, cur, used = [], [], 0
    for i, n in enumerate(lengths):
        if n == 0:
            continue
        if n > max_length:
            raise ValueError(f"sample {i} has {n} tokens, more than max_length={max_length}")
        if used + n > max_length:
            rows.append(cur)
            cur, used = [], 0
        cur.append(i)
        used += n
    if cur:
        rows.append(cur)
    return rows


class PackedSFTDataset(Dataset):
    """The prepared SFT corpus of :class:`SFTDataset`, packed into rows of ``max_length`` tokens (``position_ids``
    packing, as Hugging Face's ``position_ids`` collator, TRL's ``packing=True`` and Megatron's
    ``reset_position_ids`` / ``reset_attention_mask``).  Each sample keeps its tokens up to
    :func:`sample_length`; samples without a trainable label are dropped.  A row carries ``input_ids``, ``labels``
    (``IGNORE_INDEX`` on the padding tail; a document's last token predicts nothing, so no label crosses a document
    boundary) and ``position_ids``, which restart at 0 at every document; the padding tail counts as one more document.
    ``fill_rate`` is the share of row tokens that belong to a sample."""

    def __init__(self, path, max_length: int, tokenizer=None):
        data = torch.load(path, weights_only=False) if isinstance(path, (str, os.PathLike)) else list(path)
        self.max_length, self.tokenizer = int(max_length), tokenizer
        pad_id = getattr(tokenizer, "pad_token_id", None)
        pad_id = 0 if pad_id is None else int(pad_id)
        lengths = [sample_length(item["labels"]) for item in data]
        self.rows = []
        for members in pack_samples(lengths, self.max_length):
            ids = torch.full((self.max_length,), pad_id, dtype=torch.long)
            labels = torch.full((self.max_length,), IGNORE_INDEX, dtype=torch.long)
            pos = torch.zeros(self.max_length, dtype=torch.long)
            at = 0
            for i in members:
                n = lengths[i]
                ids[at : at + n] = torch.as_tensor(data[i]["input_ids"], dtype=torch.long)[:n]
                lab = torch.as_tensor(data[i]["labels"], dtype=torch.long)[:n].clone()
                lab[n - 1] = IGNORE_INDEX
                labels[at : at + n] = lab
                pos[at : at + n] = torch.arange(n)
                at += n
            pos[at:] = torch.arange(self.max_length - at)
            self.rows.append((ids, labels, pos))
        self.fill_rate = sum(lengths) / max(1, len(self.rows) * self.max_length)

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, index):
        ids, labels, pos = self.rows[index]
        return Instance(
            input_ids=DistTensorData(ids),
            labels=DistTensorData(labels, placement_idx=-1),
            position_ids=DistTensorData(pos),
        )


def generate_prompt(example: dict) -> str:
    """The Stanford-Alpaca prompt: instruction (+ optional input) followed by a ``### Response:`` header."""
    if example.get("input"):
        return (
            "Below is an instruction that describes a task, paired with an input that provides further context. "
            "Write a response that appropriately completes the request.\n\n"
            f"### Instruction:\n{example['instruction']}\n\n### Input:\n{example['input']}\n\n### Response:"
        )
    return (
        "Below is an instruction that describes a task. Write a response that appropriately completes the request.\n\n"
        f"### Instruction:\n{example['instruction']}\n\n### Response:"
    )


def prepare_sample(example: dict, tokenizer, max_length: int, mask_inputs: bool = True, prompt_fn=generate_prompt) -> dict:
    """``input_ids`` = ``<s> prompt response </s>`` padded to ``max_length``; ``labels`` = next-token targets with
    the prompt part (and the padding) set to ``IGNORE_INDEX``."""
    prompt_text = prompt_fn(example)
    prompt = tokenizer.tokenize(prompt_text, add_bos=True, add_eos=False, device=None)[0]
    full = tokenizer.tokenize(prompt_text + example["output"], add_bos=True, add_eos=True, device=None)[0]
    full = full[:max_length]
    labels = full.clone()
    if mask_inputs:
        labels[: min(len(prompt), len(full))] = IGNORE_INDEX
    pad = max_length - len(full)
    input_ids = torch.cat([full, torch.full((pad,), tokenizer.pad_token_id, dtype=torch.long)])
    labels = torch.cat([labels, torch.full((pad,), IGNORE_INDEX, dtype=torch.long)])
    # shift: position t predicts token t+1
    labels = torch.cat([labels[1:], torch.full((1,), IGNORE_INDEX, dtype=torch.long)])
    return {**example, "input_ids": input_ids, "labels": labels}


def prepare_sft_corpus(json_file: str, out_dir: str, tokenizer, max_seq_length: int = 512, test_split_size: int = 2000,
                       mask_inputs: bool = True, seed: int = 42, prompt_fn=generate_prompt):
    """Alpaca-format json → ``out_dir/{train,test}`` tensors files."""
    with open(json_file, "r", encoding="utf-8") as f:
        data = json.load(f)
    rng = random.Random(seed)
    rng.shuffle(data)
    test_split_size = min(test_split_size, max(1, len(data) // 10))
    test, train = data[:test_split_size], data[test_split_size:]
    os.makedirs(out_dir, exist_ok=True)
    for name, split in (("train", train), ("test", test)):
        torch.save([prepare_sample(ex, tokenizer, max_seq_length, mask_inputs, prompt_fn) for ex in split],
                   os.path.join(out_dir, name))
    return len(train), len(test)


class SentencePieceTokenizer:
    def __init__(self, pretrained_model_path, bos_token="<s>", eos_token="</s>", pad_token="<unk>", bos_token_id=None,
                 eos_token_id=None):
        import sentencepiece as spm

        self.sp_model = spm.SentencePieceProcessor()
        self.sp_model.Load(pretrained_model_path)
        self.bos_token, self.eos_token, self.pad_token = bos_token, eos_token, pad_token
        self.bos_token_id = self.sp_model.bos_id() if self.sp_model.bos_id() >= 0 else bos_token_id
        self.eos_token_id = self.sp_model.eos_id() if self.sp_model.eos_id() >= 0 else eos_token_id
        self.pad_token_id = 0
        self.eod_token = None

    @property
    def vocab_size(self):
        return self.sp_model.get_piece_size()

    def __len__(self):
        return self.vocab_size

    def padded_vocab_size(self, multiple=1):
        return (self.vocab_size + multiple - 1) // multiple * multiple

    def get_vocab(self):
        return {self.convert_id_to_token(i): i for i in range(self.vocab_size)}

    def encode(self, text, return_tensors=None, **kwargs):
        ids = self.sp_model.encode(text)
        if return_tensors in ("pt", "of"):
            return torch.tensor(ids if isinstance(text, list) else [ids], dtype=torch.long)
        return ids

    def tokenize(self, text, add_bos=False, add_eos=False, padding=False, device=None, max_length=4096, **kwargs):
        texts: List[str] = [text] if isinstance(text, str) else list(text)
        tokens = [self.sp_model.encode(s)[:max_length] for s in texts]
        if add_bos:
            tokens = [[self.bos_token_id] + t for t in tokens]
        if add_eos:
            tokens = [t + [self.eos_token_id] for t in tokens]
        if padding or len({len(t) for t in tokens}) > 1:
            width = max(len(t) for t in tokens)
            tokens = [t + (width - len(t)) * [self.pad_token_id] for t in tokens]
        out = torch.tensor(tokens, dtype=torch.long)
        if device and (device != "cuda" or torch.cuda.is_available()):
            out = out.to(device)
        return out

    def decode(self, tokens, skip_special_tokens=True, **kwargs):
        if torch.is_tensor(tokens):
            tokens = tokens.tolist()
        return self.sp_model.decode(tokens)

    def convert_token_to_id(self, token):
        return self.sp_model.piece_to_id(token)

    def convert_id_to_token(self, index):
        return self.sp_model.IdToPiece(index)


class ByteBPEChatTokenizer:
    """Byte-level BPE (``vocab.json`` + ``merges.txt``) behind the same small API as ``SentencePieceTokenizer``
    (Aquila: reference projects/Aquila/tokenizer.py; Qwen2: reference projects/Qwen/tokenizer.py).  ``special_tokens``
    are matched verbatim before BPE; ``pattern`` overrides the GPT-2 pre-tokenisation regex."""

    def __init__(self, vocab_file, merges_file, bos_token=None, eos_token="<|endoftext|>", pad_token="<|endoftext|>",
                 unk_token="<|endoftext|>", special_tokens=(), pattern=None, errors="replace"):
        import regex as re

        from libai_b200.tokenizer.tokenization_gpt2 import ByteLevelBPE

        self._bpe = ByteLevelBPE(vocab_file, merges_file, errors)
        if pattern is not None:
            self._bpe.pat = re.compile(pattern)
        self.encoder, self.decoder = self._bpe.encoder, self._bpe.decoder
        self.special = {}
        for tok in list(special_tokens) + [t for t in (bos_token, eos_token, pad_token, unk_token) if t]:
            if tok not in self.special:
                if tok not in self.encoder:
                    self.encoder[tok] = len(self.encoder)
                    self.decoder[self.encoder[tok]] = tok
                self.special[tok] = self.encoder[tok]
        self._special_re = re.compile("(" + "|".join(re.escape(t) for t in sorted(self.special, key=len, reverse=True)) + ")") \
            if self.special else None
        self.bos_token, self.eos_token, self.pad_token, self.unk_token = bos_token, eos_token, pad_token, unk_token
        self.bos_token_id = self.encoder.get(bos_token) if bos_token else None
        self.eos_token_id = self.encoder.get(eos_token) if eos_token else None
        self.pad_token_id = self.encoder.get(pad_token, 0) if pad_token else 0
        self.eod_token = None

    @property
    def vocab_size(self):
        return len(self.encoder)

    def __len__(self):
        return self.vocab_size

    def padded_vocab_size(self, multiple=1):
        return (self.vocab_size + multiple - 1) // multiple * multiple

    def get_vocab(self):
        return dict(self.encoder)

    def encode(self, text, return_tensors=None, **kwargs):
        ids = []
        chunks = self._special_re.split(text) if self._special_re is not None else [text]
        for chunk in chunks:
            if not chunk:
                continue
            if chunk in self.special:
                ids.append(self.special[chunk])
            else:
                ids.extend(self.encoder.get(t, self.encoder.get(self.unk_token, 0)) for t in self._bpe.tokenize(chunk))
        if return_tensors in ("pt", "of"):
            return torch.tensor([ids], dtype=torch.long)
        return ids

    def tokenize(self, text, add_bos=False, add_eos=False, padding=False, device=None, max_length=4096, **kwargs):
        texts = [text] if isinstance(text, str) else list(text)
        tokens = [self.encode(s)[:max_length] for s in texts]
        if add_bos and self.bos_token_id is not None:
            tokens = [[self.bos_token_id] + t for t in tokens]
        if add_eos and self.eos_token_id is not None:
            tokens = [t + [self.eos_token_id] for t in tokens]
        if padding or len({len(t) for t in tokens}) > 1:
            width = max(len(t) for t in tokens)
            tokens = [t + (width - len(t)) * [self.pad_token_id] for t in tokens]
        out = torch.tensor(tokens, dtype=torch.long)
        if device and (device != "cuda" or torch.cuda.is_available()):
            out = out.to(device)
        return out

    def decode(self, tokens, skip_special_tokens=True, **kwargs):
        if torch.is_tensor(tokens):
            tokens = tokens.tolist()
        pieces, run = [], []
        special_ids = set(self.special.values())
        for t in tokens:
            if t in special_ids:
                if run:
                    pieces.append(self._bpe.detokenize(run))
                    run = []
                if not skip_special_tokens:
                    pieces.append(self.decoder[t])
            else:
                run.append(self.decoder.get(t, ""))
        if run:
            pieces.append(self._bpe.detokenize(run))
        return "".join(pieces)

    def convert_token_to_id(self, token):
        return self.encoder.get(token)

    def convert_id_to_token(self, index):
        return self.decoder.get(index)
