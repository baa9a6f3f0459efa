"""Token constraints of ``generate()``: ``no_repeat_ngram_size``, ``sequence_bias``, ``bad_words_ids``, ``min_length`` /
``min_new_tokens``, ``suppress_tokens`` and ``begin_suppress_tokens`` with transformers 5.5's meanings
(hf:generation/logits_process.py and utils.py ``_get_logits_processor`` / ``_prepare_generated_length``).

``LogitsConstraints.build`` checks the arguments where HF's processor constructors do and packs them into the table
``uvx_logits_constraints`` reads (include/uvx.h): one entry per (token sequence, bias, kind), a token's entries consecutive in
HF's order, so that the kernel's one thread per token adds and sets exactly what HF's processors do, one after the other."""
from __future__ import annotations

import dataclasses
import numbers
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

CK_BIAS, CK_BAD, CK_SUPPRESS, CK_BEGIN, CK_MIN_LEN = 0, 1, 2, 3, 4     # UVX_CK_* (include/uvx.h)


def _is_int(x) -> bool:
    return isinstance(x, (int, np.integer))


def _ngram(n) -> int:
    """HF builds NoRepeatNGramLogitsProcessor only for n > 0 (anything else is ignored), and its constructor wants a Python
    int."""
    if n is None:
        return 0
    try:
        on = bool(n > 0)
    except TypeError:
        raise ValueError(f"`no_repeat_ngram_size` has to be a strictly positive integer, but is {n}") from None
    if not on:
        return 0
    if not isinstance(n, int):
        raise ValueError(f"`ngram_size` has to be a strictly positive integer, but is {n}")
    return int(n)


def _min_count(name: str, v) -> Optional[int]:
    if v is None:
        return None
    if not _is_int(v):
        raise ValueError(f"`{name}` has to be a non-negative integer, but is {v}")
    return int(v)


def _sequence_bias(sequence_bias) -> List[Tuple[Tuple[int, ...], float]]:
    """HF's ``SequenceBiasLogitsProcessor._validate_arguments`` + ``_convert_list_arguments_into_dict``: the list form
    ``[[ids], float]`` (ids > 0) or the dict form ``{tuple: float}`` (ids >= 0) -> (ids, bias) in dict order (a later duplicate
    overwrites an earlier one and keeps its place)."""
    if not isinstance(sequence_bias, (dict, list)) or len(sequence_bias) == 0:
        raise ValueError(f"`sequence_bias` has to be a non-empty dictionary, or non-empty list of lists but is {sequence_bias}.")
    if isinstance(sequence_bias, dict):
        for ids, b in sequence_bias.items():
            if not isinstance(ids, tuple) or len(ids) == 0 or any(not _is_int(t) or t < 0 for t in ids):
                raise ValueError(f"Each key in `sequence_bias` has to be a non-empty tuple of positive integers, but is "
                                 f"{sequence_bias}.")
            if not isinstance(b, float):
                raise ValueError(f"`sequence_bias` has to be a dict with floats as values, but is {sequence_bias}.")
        items = list(sequence_bias.items())
    else:
        for e in sequence_bias:
            ok = isinstance(e, (list, tuple)) and len(e) == 2 and isinstance(e[0], list) and len(e[0]) > 0 and \
                all(_is_int(t) and t > 0 for t in e[0]) and isinstance(e[1], float)
            if not ok:
                raise ValueError(f"Each element in `sequence_bias` has to be a non-empty list of lists of positive integers "
                                 f"and float, but is {sequence_bias}.")
        items = [(tuple(e[0]), e[1]) for e in sequence_bias]
    merged = {}
    for ids, b in items:
        merged[tuple(int(t) for t in ids)] = float(b)
    return list(merged.items())


def _bad_words(bad_words_ids, eos: Sequence[int]) -> List[Tuple[int, ...]]:
    """HF's ``NoBadWordsLogitsProcessor``: checks, single-token entries equal to an EOS id dropped, duplicates merged."""
    if not isinstance(bad_words_ids, list) or len(bad_words_ids) == 0:
        raise ValueError(f"`bad_words_ids` has to be a non-empty list, but is {bad_words_ids}.")
    if any(not isinstance(w, list) for w in bad_words_ids):
        raise ValueError(f"`bad_words_ids` has to be a list of lists, but is {bad_words_ids}.")
    if any(any(not _is_int(t) or t < 0 for t in w) for w in bad_words_ids):
        raise ValueError(f"Each list in `bad_words_ids` has to be a list of positive integers, but is {bad_words_ids}.")
    words = [w for w in bad_words_ids if all(w != [e] for e in eos)]
    if any(len(w) == 0 for w in words):
        raise ValueError(f"Each list in `bad_words_ids` has to be a non-empty list of positive integers, but is {bad_words_ids}.")
    return list(dict.fromkeys(tuple(int(t) for t in w) for w in words))


def _token_list(name: str, tokens) -> List[int]:
    if tokens is None:
        return []
    tokens = list(tokens)
    if any(not _is_int(t) for t in tokens):
        raise ValueError(f"`{name}` has to be a list of integers, but is {tokens}")
    return [int(t) for t in tokens]


@dataclasses.dataclass
class LogitsConstraints:
    """One request's constraints as the kernel reads them: ``ngram`` (0: off), ``min_len`` (EOS ids are banned while the
    sequence is shorter), ``begin_len`` (the sequence length at the first new token) and ``entries`` in table order, each
    (ids, bias, kind) with the target token last."""
    ngram: int
    min_len: int
    begin_len: int
    entries: List[Tuple[Tuple[int, ...], float, int]]

    @classmethod
    def build(cls, vocab_size: int, eos: Sequence[int], prompt_len: int, no_repeat_ngram_size=None, bad_words_ids=None,
              sequence_bias=None, min_length=None, min_new_tokens=None, suppress_tokens=None,
              begin_suppress_tokens=None) -> Optional["LogitsConstraints"]:
        """The constraints of a call whose prompt (the whole ``input_ids``, earlier turns included) has ``prompt_len`` tokens, or
        None when none applies.  ValueError where HF's constructors raise, and for ids >= ``vocab_size`` in ``sequence_bias``
        / ``bad_words_ids`` (HF's ``_prepare_bias_variables``)."""
        V, S = int(vocab_size), int(prompt_len)
        eos = [int(e) for e in eos]
        ngram = _ngram(no_repeat_ngram_size)
        min_length, min_new = _min_count("min_length", min_length), _min_count("min_new_tokens", min_new_tokens)
        bias = _sequence_bias(sequence_bias) if sequence_bias is not None else []
        bad = _bad_words(bad_words_ids, eos) if bad_words_ids is not None else []
        too_big = [t for ids in [b[0] for b in bias] + bad for t in ids if t >= V]
        if too_big:
            raise ValueError(f"The model vocabulary size is {V}, but the following tokens were being biased: {too_big}")
        suppress = _token_list("suppress_tokens", suppress_tokens)
        begin = _token_list("begin_suppress_tokens", begin_suppress_tokens)
        # _prepare_generated_length: min_new_tokens, when given, replaces min_length by prompt length + min_new_tokens; both
        # processors then ban EOS while the sequence is shorter than that (and only when EOS ids are set)
        min_len = S + min_new if min_new is not None else (min_length or 0)
        if not eos or min_len <= 0:
            min_len = 0
        rows = []       # (target, rank, order, ids, bias, kind): sorted, a token's entries in HF's order
        for i, (ids, b) in enumerate(bias):
            rows.append((ids[-1], 0 if len(ids) == 1 else 1, i, ids, b, CK_BIAS))
        for i, ids in enumerate(bad):
            rows.append((ids[-1], 2, i, ids, float("-inf"), CK_BAD))
        for kind, toks in ((CK_SUPPRESS, suppress), (CK_BEGIN, begin), (CK_MIN_LEN, eos if min_len else [])):
            for t in dict.fromkeys(toks):
                if 0 <= t < V:          # any other id never matches a vocabulary entry
                    rows.append((t, 3, kind, (t,), 0.0, kind))
        if not rows and ngram == 0:
            return None
        rows.sort(key=lambda r: r[:3])
        return cls(ngram, min_len, S, [(r[3], r[4], r[5]) for r in rows])

    @property
    def n_ids(self) -> int:
        """Table size in ids (what a slot's ``max_constraint_tokens`` must cover)."""
        return sum(len(e[0]) for e in self.entries)

    def tables(self, width: Optional[int] = None):
        """(cfg int32 [4], ids int64 [T], end int32 [T], bias fp32 [T], kind int32 [T]) numpy arrays, T = ``width`` (default
        the table's id count, at least 1; unused entries are zero)."""
        T = max(1, self.n_ids) if width is None else int(width)
        if self.n_ids > T:
            raise ValueError(f"the constraints need a table of {self.n_ids} ids; this one holds {T}")
        ids = np.zeros(T, np.int64)
        end = np.zeros(T, np.int32)
        bias = np.zeros(T, np.float32)
        kind = np.zeros(T, np.int32)
        o = 0
        for j, (e_ids, b, k) in enumerate(self.entries):
            ids[o:o + len(e_ids)] = e_ids
            o += len(e_ids)
            end[j], bias[j], kind[j] = o, np.float32(b), k
        cfg = np.array([self.ngram, self.min_len, self.begin_len, len(self.entries)], np.int32)
        return cfg, ids, end, bias, kind

    def device_tables(self, device) -> Tuple[torch.Tensor, ...]:
        """``tables()`` as device tensors, the argument of ``ops.logits_constraints_``."""
        return tuple(torch.from_numpy(a).to(device) for a in self.tables())
