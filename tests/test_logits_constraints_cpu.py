"""Host side of the token constraints (ultravox_b200/constraints.py): the packed table walked by a numpy restatement of the
kernel's rule (include/uvx.h uvx_logits_constraints) equals transformers' processors, and the argument checks raise where
transformers' constructors do.  No GPU needed."""
import pathlib
import re

import numpy as np
import pytest
import torch
from transformers.generation import logits_process as lp

from ultravox_b200 import _lib
from ultravox_b200.constraints import CK_BAD, CK_BEGIN, CK_BIAS, CK_MIN_LEN, CK_SUPPRESS, LogitsConstraints

ROOT = pathlib.Path(__file__).resolve().parents[1]


@np.errstate(invalid="ignore")        # inf - inf biases make NaN on purpose
def walk(c: LogitsConstraints, x: np.ndarray, seq: np.ndarray) -> np.ndarray:
    """uvx_logits_constraints on one fp32 row x over seq[0:L], from the packed table (include/uvx.h)."""
    cfg, ids, end, bias, kind = c.tables()
    n, min_len, begin_len, n_ent = (int(v) for v in cfg)
    L, V = len(seq), len(x)
    x = x.copy()
    for e in range(n_ent):
        t = ids[end[e] - 1]
        if e > 0 and ids[end[e - 1] - 1] == t:
            continue
        sb, bw = np.float32(0), np.float32(0)
        has_sb = has_bw = hit = False
        j = e
        while j < n_ent and ids[end[j] - 1] == t:
            lo, hi = (end[j - 1] if j else 0), end[j]
            k, ln = kind[j], hi - lo
            has_sb |= k == CK_BIAS
            has_bw |= k == CK_BAD
            if ln <= L and all(seq[L - ln + 1 + i] == ids[lo + i] for i in range(ln - 1)):
                if k == CK_BIAS:
                    sb = np.float32(sb + bias[j])
                elif k == CK_BAD:
                    bw = np.float32(bw + bias[j])
                else:
                    hit |= k == CK_SUPPRESS or (k == CK_BEGIN and L == begin_len) or (k == CK_MIN_LEN and L < min_len)
            j += 1
        v = x[t]
        if has_sb:
            v = np.float32(v + sb)
        if has_bw:
            v = np.float32(v + bw)
        x[t] = -np.inf if hit else v
    if n >= 1 and L + 1 >= n:
        for e in range(n - 1, L):
            if all(seq[e - i] == seq[L - i] for i in range(1, n)):
                x[seq[e]] = -np.inf
    return x


def hf_processors(V, eos, S, no_repeat_ngram_size=None, bad_words_ids=None, sequence_bias=None, min_length=None,
                  min_new_tokens=None, suppress_tokens=None, begin_suppress_tokens=None):
    """transformers' processor list in _get_logits_processor's order, with _prepare_generated_length's min_length."""
    eos_t = torch.tensor(eos) if eos else None
    if min_new_tokens is not None:
        min_length = min_new_tokens + S
    procs = []
    if sequence_bias is not None:
        procs.append(lp.SequenceBiasLogitsProcessor(sequence_bias=sequence_bias))
    if no_repeat_ngram_size is not None and no_repeat_ngram_size > 0:
        procs.append(lp.NoRepeatNGramLogitsProcessor(no_repeat_ngram_size))
    if bad_words_ids is not None:
        procs.append(lp.NoBadWordsLogitsProcessor(bad_words_ids, eos_t))
    if min_length is not None and eos_t is not None and min_length > 0:
        procs.append(lp.MinLengthLogitsProcessor(min_length, eos_t))
    if min_new_tokens is not None and eos_t is not None and min_new_tokens > 0:
        procs.append(lp.MinNewTokensLengthLogitsProcessor(S, min_new_tokens, eos_t))
    if suppress_tokens is not None:
        procs.append(lp.SuppressTokensLogitsProcessor(suppress_tokens))
    if begin_suppress_tokens is not None:
        procs.append(lp.SuppressTokensAtBeginLogitsProcessor(begin_suppress_tokens, S))
    return procs


def hf_apply(procs, x: np.ndarray, seq: np.ndarray) -> np.ndarray:
    s = torch.from_numpy(x.copy())[None]
    ids = torch.from_numpy(seq.astype(np.int64))[None]
    for p in procs:
        s = p(ids, s)
    return s[0].numpy()


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def test_abi_symbols_bound():
    header = (ROOT / "include" / "uvx.h").read_text()
    names = [n for n in re.findall(r"\b(uvx_logits_constraints[a-z_]*)\s*\(", header)]
    assert sorted(set(names)) == ["uvx_logits_constraints", "uvx_logits_constraints_rows", "uvx_logits_constraints_rows_map",
                                  "uvx_logits_constraints_slots"]
    for name in names:
        assert name in _lib.SIGNATURES, name
    lib = _lib.lib()
    for name in names:
        assert hasattr(lib, name), name
    consts = dict(re.findall(r"#define (UVX_CK_[A-Z_]+) (\d+)", header))
    assert consts == {"UVX_CK_BIAS": str(CK_BIAS), "UVX_CK_BAD": str(CK_BAD), "UVX_CK_SUPPRESS": str(CK_SUPPRESS),
                      "UVX_CK_BEGIN": str(CK_BEGIN), "UVX_CK_MIN_LEN": str(CK_MIN_LEN)}


def test_sequence_bias_dict_order_and_duplicates():
    # list form: the later [[5], ...] overwrites the earlier one but keeps its place ahead of [[3, 5], ...]
    sb = [[[5], 1.5], [[3, 5], 0.25], [[5], -2.0], [[7, 3, 5], 1e30], [[3, 5], 3.0]]
    c = LogitsConstraints.build(16, [], 4, sequence_bias=sb)
    targets5 = [e for e in c.entries if e[0][-1] == 5]
    assert [e[0] for e in targets5] == [(5,), (3, 5), (7, 3, 5)]
    assert [e[1] for e in targets5] == [-2.0, 3.0, 1e30]


def test_bad_words_drop_eos_singles_only():
    c = LogitsConstraints.build(16, [2, 9], 3, bad_words_ids=[[2], [9], [4, 2], [6], [6], [2, 9, 9]])
    assert [e[0] for e in c.entries] == [(4, 2), (6,), (2, 9, 9)]
    assert all(e[2] == CK_BAD and e[1] == float("-inf") for e in c.entries)
    assert LogitsConstraints.build(16, [2], 3, bad_words_ids=[[2]]) is None      # everything was an EOS id


def test_entries_longer_than_sequence_skipped():
    c = LogitsConstraints.build(16, [], 2, sequence_bias={(1, 2, 3): 5.0, (3,): 1.0}, bad_words_ids=[[1, 2, 3, 4]])
    x = np.arange(16, dtype=np.float32)
    seq = np.array([1, 2])
    out = walk(c, x, seq)
    assert _same(out, hf_apply(hf_processors(16, [], 2, sequence_bias={(1, 2, 3): 5.0, (3,): 1.0},
                                              bad_words_ids=[[1, 2, 3, 4]]), x, seq))
    assert out[3] == 4.0 and out[4] == 4.0


@pytest.mark.parametrize("seed", range(40))
def test_table_walk_equals_hf(seed):
    rng = np.random.default_rng(seed)
    V = int(rng.choice([12, 40, 200]))
    L = int(rng.integers(1, 60))
    S = int(rng.integers(1, L + 1))
    seq = rng.integers(0, min(V, 8), size=L)       # a small alphabet: repeats, matches and overlaps are common
    eos = sorted(set(int(e) for e in rng.integers(0, V, size=int(rng.integers(0, 3)))))
    kw = {}
    if rng.random() < 0.6:
        kw["no_repeat_ngram_size"] = int(rng.integers(1, 6))
    if rng.random() < 0.6:
        items = []
        for _ in range(int(rng.integers(1, 8))):
            ids = [int(t) for t in rng.integers(1, min(V, 8), size=int(rng.integers(1, 4)))]
            b = float(rng.choice([rng.normal() * 3, float("-inf"), float("inf"), 0.5]))
            items.append([ids, b])
        kw["sequence_bias"] = items
    if rng.random() < 0.5:
        kw["bad_words_ids"] = [[int(t) for t in rng.integers(0, min(V, 8), size=int(rng.integers(1, 4)))]
                               for _ in range(int(rng.integers(1, 6)))]
    if rng.random() < 0.4:
        kw["min_length"] = int(rng.integers(0, L + 3))
    if rng.random() < 0.4:
        kw["min_new_tokens"] = int(rng.integers(0, L - S + 3))
    if rng.random() < 0.4:
        kw["suppress_tokens"] = [int(t) for t in rng.integers(0, V, size=3)]
    if rng.random() < 0.4:
        kw["begin_suppress_tokens"] = [int(t) for t in rng.integers(0, V, size=3)]
    x = (rng.standard_normal(V) * 4).astype(np.float32)
    x[rng.integers(0, V, size=3)] = [np.inf, -np.inf, np.nan]
    for L_now in {L, S}:       # the first new token (L == S) and a later one
        s_now = seq[:L_now]
        c = LogitsConstraints.build(V, eos, S, **kw)
        want = hf_apply(hf_processors(V, eos, S, **kw), x, s_now)
        got = x.copy() if c is None else walk(c, x, s_now)
        assert _same(got, want), (kw, L_now)


@pytest.mark.parametrize("kw", [
    dict(bad_words_ids=[1, 2]), dict(bad_words_ids=[]), dict(bad_words_ids=[[1, -2]]), dict(bad_words_ids=[[1.0]]),
    dict(bad_words_ids=[[]]), dict(sequence_bias=[[[1], 1]]), dict(sequence_bias=[[[0], 1.0]]), dict(sequence_bias={}),
    dict(sequence_bias={(1,): 1}), dict(sequence_bias={(-1,): 1.0}), dict(sequence_bias={(): 1.0}),
    dict(sequence_bias={1: 1.0}), dict(no_repeat_ngram_size=2.0), dict(min_length=3.5), dict(min_new_tokens="2"),
])
def test_validation_matches_hf(kw):
    with pytest.raises(ValueError):
        LogitsConstraints.build(32, [0], 4, **kw)
    # transformers rejects the same arguments (an empty bad word only once the processor runs)
    with pytest.raises((ValueError, TypeError, IndexError)):
        for p in hf_processors(32, [0], 4, **kw):
            p(torch.zeros(1, 4, dtype=torch.long), torch.zeros(1, 32))


def test_ngram_size_edges_follow_hf():
    # HF builds the processor only for n > 0 (anything else is ignored) and its constructor takes Python ints only
    for n in (0, -1, 0.0, -1.5):
        assert LogitsConstraints.build(32, [], 4, no_repeat_ngram_size=n) is None
    for n in (2.0, np.int64(2)):
        with pytest.raises(ValueError):
            LogitsConstraints.build(32, [], 4, no_repeat_ngram_size=n)
        with pytest.raises(ValueError):
            lp.NoRepeatNGramLogitsProcessor(n)


def test_ids_outside_vocabulary_raise():
    with pytest.raises(ValueError, match="vocabulary size"):
        LogitsConstraints.build(32, [], 4, sequence_bias={(40,): 1.0})
    with pytest.raises(ValueError, match="vocabulary size"):
        LogitsConstraints.build(32, [], 4, bad_words_ids=[[3, 32]])


def test_nothing_to_do_is_none_and_table_width():
    assert LogitsConstraints.build(32, [1], 4) is None
    assert LogitsConstraints.build(32, [], 4, min_new_tokens=3) is None          # no EOS ids: HF adds no processor
    assert LogitsConstraints.build(32, [1], 4, no_repeat_ngram_size=0) is None
    c = LogitsConstraints.build(32, [1], 4, bad_words_ids=[[3, 4, 5]], min_new_tokens=2)
    assert c.n_ids == 4 and c.min_len == 6
    assert c.tables(8)[1].shape == (8,)
    with pytest.raises(ValueError):
        c.tables(3)
