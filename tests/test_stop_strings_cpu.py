"""Stop strings on the host: the packed sparse table of ultravox_b200.stop_strings, walked by its numpy rule, against transformers'
own StopStringCriteria.__call__ on random and constructed sequences (byte-level and Metaspace vocabularies, V = 1024 and
128256), the argument checks of generate() / submit(), and the new ABI symbols."""
import ctypes
import os

import numpy as np
import pytest
import torch

from ultravox_b200 import stop_strings as ss

V8B = 128256
_ALPHA = "abcdefghijklmnopqrstuvwxyz:.,!?\n"


def make_tokenizer(V: int, kind: str = "bytelevel", seed: int = 0):
    """A PreTrainedTokenizerFast over an in-memory BPE vocabulary of exactly V ids: every single character of a small alphabet,
    then distinct random 2-6 character pieces, each optionally with the word-start mark (Ġ byte-level, ▁ Metaspace)."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    mark = "Ġ" if kind == "bytelevel" else "▁"
    nl = "Ċ" if kind == "bytelevel" else "\n"
    chars = [c if c != "\n" else nl for c in _ALPHA] + [mark]
    if kind == "bytelevel":
        chars = sorted(set(chars) | set(pre_tokenizers.ByteLevel.alphabet()))
    rng = np.random.default_rng(seed)
    vocab = {c: i for i, c in enumerate(dict.fromkeys(chars))}
    pieces = [c for c in chars if c not in (mark,)]
    while len(vocab) < V:
        n = int(rng.integers(2, 7))
        t = "".join(rng.choice(pieces[:len(_ALPHA)], size=n))
        if rng.random() < 0.4:
            t = mark + t
        vocab.setdefault(t, len(vocab))
    tk = Tokenizer(models.BPE(vocab=vocab, merges=[]))
    if kind == "bytelevel":
        tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
        tk.decoder = decoders.ByteLevel()
    else:
        tk.pre_tokenizer = pre_tokenizers.Metaspace(replacement=mark, prepend_scheme="never")
        tk.decoder = decoders.Metaspace(replacement=mark, prepend_scheme="never")
    return PreTrainedTokenizerFast(tokenizer_object=tk)


def hf_hits(crit, seqs) -> list:
    return [bool(h) for h in crit(torch.as_tensor(np.asarray(seqs, dtype=np.int64)), None)]


def _check(tok, strings, seqs):
    st = ss.StopStrings.build(tok, strings)
    want = hf_hits(st.criteria, seqs)
    got = [ss.walk(st.table, s) for s in seqs]
    assert got == want, (strings, got, want)
    return sum(want)


def _text_ids(tok, text):
    return tok(text, add_special_tokens=False)["input_ids"]


@pytest.mark.parametrize("kind", ["bytelevel", "metaspace"])
@pytest.mark.parametrize("V", [1024, V8B])
def test_walk_equals_hf(kind, V):
    tok = make_tokenizer(V, kind, seed=V % 7)
    rng = np.random.default_rng(V + len(kind))
    text = " the user: hello there.\nuser: fine, ok! assistant: done."
    ids = _text_ids(tok, text)
    dec = tok.decode(ids)
    hits = 0
    sets = [["user:"], ["r: f", "ok!", ".\n"], ["user", "user:", "er"], ["abab", "baba", "ab"], ["e", ":", "hello there"],
            [dec[5:17], dec[-9:], "!", "ne.", dec[20:23]]]
    for strings in sets:
        seqs = [ids[:L] for L in range(1, len(ids) + 1)]
        # random ids, ids outside the tokenizer's table, and constructed ends
        for L in (1, 2, 5, 40):
            seqs.append(list(rng.integers(0, V, size=L)))
        seqs.append(ids[:6] + [V + 5])
        seqs.append([V + 7] + ids[:9])
        L0 = max(len(s) for s in seqs)
        padded = [[0] * (L0 - len(s)) + list(s) for s in seqs]          # HF's call takes one rectangular batch
        hits += _check(tok, strings, padded)
        for s in seqs[:8]:
            hits += _check(tok, strings, [s])
    assert hits > 10


def test_table_is_sparse_and_cached():
    tok = make_tokenizer(V8B, "bytelevel", seed=3)
    a = ss.StopStrings.build(tok, ["\nUser:", "stop"])
    emb = a.criteria.embedding_vec
    assert a.n_words < emb.numel() // 4
    n_ent, n_stop, mvp, mvel, wmax = a.table[:5].tolist()
    assert n_stop == 2 and wmax == 6 and 0 < n_ent < V8B
    ids = a.table[5 + n_stop:5 + n_stop + n_ent]
    assert (np.diff(ids) > 0).all()
    b = ss.StopStrings.build(tok, ["\nUser:", "stop"])
    assert b is a                                # built once per (tokenizer, strings)


def test_argument_errors():
    tok = make_tokenizer(1024, "metaspace")
    assert ss.StopStrings.build(tok, None) is None and ss.StopStrings.build(None, None) is None
    with pytest.raises(ValueError, match="tokenizer"):
        ss.StopStrings.build(None, "stop")
    for bad in ("", ["a", ""], []):
        with pytest.raises(ValueError):
            ss.StopStrings.build(tok, bad)
    for bad in (5, ["a", 3], b"ab"):
        with pytest.raises(TypeError):
            ss.StopStrings.build(tok, bad)
    with pytest.raises(ValueError):             # no vocabulary token can end it: HF's constructor raises
        ss.StopStrings.build(tok, "€")
    assert ss.StopStrings.build(tok, "ab").stop_strings == ("ab",)


def test_abi_symbols_present():
    so = os.path.join(os.path.dirname(ss.__file__), "libuvx.so")
    if not os.path.exists(so):
        pytest.skip("libuvx.so is not built")
    lib = ctypes.CDLL(so)
    for name in ("uvx_stop_strings", "uvx_stop_strings_slots", "uvx_stop_strings_rows", "uvx_stop_strings_rows_map",
                 "uvx_stop_strings_beam", "uvx_token_finish_stop", "uvx_slot_finish_stop", "uvx_lookup_accept_stop",
                 "uvx_lookup_accept_slots_stop", "uvx_beam_update_stop"):
        assert hasattr(lib, name), name
