"""Stop strings of ``generate()``: ``stop_strings=`` with ``tokenizer=``, with transformers 5.5's meaning
(hf:generation/stopping_criteria.py ``StopStringCriteria``).

``StopStrings.build`` constructs HF's own criteria object, so HF's vocabulary cleaning, its checks and its LRU cache of the
precompute hold as they are, and packs its dense ``embedding_vec`` [vocab + 2, n_stop * (mvp + mvel) + 1] into the sparse table
``uvx_stop_strings`` reads (include/uvx.h): only the tokens with some valid position or end overlap take part in a match, so
only their rows are kept, behind their sorted ids and a small header.  A build is cached per (tokenizer, stop strings) and
``device_table`` uploads a table once per device."""
from __future__ import annotations

import collections
from typing import Optional, Sequence, Union

import numpy as np
import torch

HEADER = 5          # n_ent, n_stop, mvp, mvel, W_max (kStopHdr in generate.cu), then the n_stop target lengths

# (id of the tokenizer, its length, stop strings) -> (tokenizer, StopStrings).  HF's own cache is keyed on the order of
# get_vocab(), which a fast tokenizer does not keep from call to call, so the same request would rebuild HF's precompute
# (seconds at V = 128k); the entry keeps the tokenizer alive, so its id stays unique
_BUILT: "collections.OrderedDict[tuple, tuple]" = collections.OrderedDict()
_TABLES_MAX = 8
_DEVICE: "collections.OrderedDict[tuple, torch.Tensor]" = collections.OrderedDict()


def check_stop_strings(stop_strings) -> Optional[tuple]:
    """``stop_strings`` as a tuple of str (None: off); ValueError for an empty list or an empty string, TypeError otherwise
    unless a str or a list / tuple of str."""
    if stop_strings is None:
        return None
    if isinstance(stop_strings, str):
        stop_strings = [stop_strings]
    if not isinstance(stop_strings, (list, tuple)) or not all(isinstance(s, str) for s in stop_strings):
        raise TypeError(f"stop_strings must be a str or a list of str, got {stop_strings!r}")
    if len(stop_strings) == 0:
        raise ValueError("stop_strings must hold at least one string")
    if any(len(s) == 0 for s in stop_strings):
        raise ValueError("stop_strings must not contain an empty string (it would match every sequence)")
    return tuple(stop_strings)


def pack(embedding_vec: np.ndarray, max_valid_positions: int, max_valid_end_lens: int, target_lens: Sequence[int]) -> np.ndarray:
    """HF's dense precompute -> the sparse int32 table: header (n_ent, n_stop, mvp, mvel, W_max), target lengths [n_stop], the
    sorted ids [n_ent] of the tokens with an entry other than -1 outside the length column, then their HF rows
    [n_ent, n_stop * (mvp + mvel) + 1] (positions of string s at s * mvp, end overlaps at n_stop * mvp + s * mvel, the token's
    length last).  HF's dummy last row (ids past its table are clamped onto it) has no entries, so it is never kept."""
    emb = np.asarray(embedding_vec, dtype=np.int32)
    n_stop = len(target_lens)
    width = n_stop * (max_valid_positions + max_valid_end_lens) + 1
    if emb.ndim != 2 or emb.shape[1] != width:
        raise ValueError(f"embedding_vec has shape {emb.shape}; expected [*, {width}]")
    ids = np.flatnonzero((emb[:, :-1] != -1).any(axis=1)).astype(np.int32)
    tl = np.asarray(target_lens, dtype=np.int32)
    head = np.array([ids.size, n_stop, max_valid_positions, max_valid_end_lens, int(tl.max())], dtype=np.int32)
    return np.concatenate([head, tl, ids, emb[ids].reshape(-1)])


class StopStrings:
    """HF's ``StopStringCriteria(tokenizer, stop_strings)`` and its sparse table (``table``, int32 numpy, ``n_words`` long)."""

    def __init__(self, criteria, table: np.ndarray):
        self.criteria = criteria
        self.stop_strings = tuple(criteria.stop_strings)
        self.table = table
        self.n_words = int(table.size)

    @classmethod
    def build(cls, tokenizer, stop_strings: Union[str, Sequence[str], None]) -> Optional["StopStrings"]:
        """None without ``stop_strings`` (a ``tokenizer`` alone is ignored, as in HF).  ValueError without a tokenizer (HF's
        message), for an empty string or list, and where HF's constructor raises (no vocabulary token can end a string)."""
        strings = check_stop_strings(stop_strings)
        if strings is None:
            return None
        if tokenizer is None:
            raise ValueError("There are one or more stop strings, either in the arguments to `generate` or in the model's "
                             "generation config, but we could not locate a tokenizer. When generating with stop strings, you "
                             "must pass the model's tokenizer to the `tokenizer` argument of `generate`.")
        key = (id(tokenizer), len(tokenizer), strings)
        hit = _BUILT.get(key)
        if hit is not None and hit[0] is tokenizer:
            _BUILT.move_to_end(key)
            return hit[1]
        from transformers.generation.stopping_criteria import StopStringCriteria
        crit = StopStringCriteria(tokenizer, list(strings))
        out = cls(crit, pack(crit.embedding_vec.numpy(), crit.max_valid_positions, crit.max_valid_end_lens,
                             crit.target_lens.tolist()))
        _BUILT[key] = (tokenizer, out)
        if len(_BUILT) > _TABLES_MAX:
            _BUILT.popitem(last=False)
        return out

    def device_table(self, device) -> torch.Tensor:
        """The table as an int32 device tensor, uploaded once per (table, device) and then reused."""
        dev = torch.device(device)
        key = (id(self.table), str(dev))
        t = _DEVICE.get(key)
        if t is None or t[0] is not self.table:
            t = (self.table, torch.from_numpy(self.table).to(dev))
            _DEVICE[key] = t
            if len(_DEVICE) > _TABLES_MAX:
                _DEVICE.popitem(last=False)
        else:
            _DEVICE.move_to_end(key)
        return t[1]


def walk(table: np.ndarray, x: Sequence[int]) -> bool:
    """The rule ``uvx_stop_strings`` runs, on the host: whether the sequence x (its last element the candidate token) ends a
    stop string, read from the packed table.  The reference the kernel is tested against, itself tested against HF's
    ``StopStringCriteria.__call__``."""
    t = np.asarray(table, dtype=np.int64)
    n_ent, n_stop, mvp, mvel, wmax = (int(v) for v in t[:HEADER])
    tgt = t[HEADER:HEADER + n_stop]
    ids = t[HEADER + n_stop:HEADER + n_stop + n_ent]
    rw = n_stop * (mvp + mvel) + 1
    rows = t[HEADER + n_stop + n_ent:].reshape(n_ent, rw) if n_ent else np.zeros((0, rw), np.int64)

    def find(tok: int) -> int:
        i = int(np.searchsorted(ids, tok))
        return i if i < n_ent and ids[i] == tok else -1

    L = len(x)
    if L == 0 or n_ent == 0:
        return False
    W = min(wmax, L)
    first = find(int(x[-1]))
    if first < 0:
        return False
    for s in range(n_stop):
        for e in rows[first, n_stop * mvp + s * mvel:n_stop * mvp + (s + 1) * mvel]:
            c = int(e)
            if c <= 0:
                continue
            if c >= tgt[s]:
                return True
            for j in range(1, W):
                y = find(int(x[L - 1 - j]))
                if y < 0 or c not in rows[y, s * mvp:(s + 1) * mvp]:
                    break
                c += int(rows[y, -1])
                if c >= tgt[s]:
                    return True
    return False
