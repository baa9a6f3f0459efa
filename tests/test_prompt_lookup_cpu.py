"""Prompt lookup decoding without a GPU: the new C ABI entries are exported and declared, and generate()'s prompt-lookup
argument checks (which run before any device work) raise what transformers raises."""
import ctypes
import pathlib
import re

import pytest
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
NEW = ("uvx_lookup_draft", "uvx_lookup_accept", "uvx_repetition_penalty_rows", "uvx_record_scores_rows")


def test_lookup_symbols_declared_bound_and_exported():
    from ultravox_b200 import _lib
    header = (ROOT / "include" / "uvx.h").read_text()
    for name in NEW:
        assert re.search(rf"\bint {name}\(", header), name
        assert name in _lib.SIGNATURES, name
    if not _lib.LIB_PATH.exists():
        pytest.skip("libuvx.so not built")
    handle = ctypes.CDLL(str(_lib.LIB_PATH))
    for name in NEW:
        assert hasattr(handle, name), name


def _check(ids, k=4, n=None, mask=None, beams=1):
    from ultravox_b200.model import UltravoxModel
    return UltravoxModel._check_lookup(ids, mask, beams, k, n)


def test_lookup_argument_checks():
    ids = torch.zeros(1, 6, dtype=torch.int64)
    assert _check(ids) == (4, 2)                        # n defaults to 2, as HF's `max_matching_ngram_size or 2`
    assert _check(ids, k=1, n=1) == (1, 1)
    assert _check(ids, k=31, n=7) == (31, 7)
    assert _check(ids, mask=torch.ones(1, 6)) == (4, 2)
    for k in (0, 32, -1, 2.0, True):
        with pytest.raises(ValueError, match="prompt_lookup_num_tokens"):
            _check(ids, k=k)
    for n in (0, -3, 1.5, False):
        with pytest.raises(ValueError, match="max_matching_ngram_size"):
            _check(ids, n=n)
    with pytest.raises(ValueError, match="assisted generate is only supported for batch_size = 1"):
        _check(torch.zeros(2, 6, dtype=torch.int64))
    with pytest.raises(ValueError, match="num_beams"):
        _check(ids, beams=2)
    mask = torch.ones(1, 6, dtype=torch.int64)
    mask[0, :2] = 0
    with pytest.raises(NotImplementedError):
        _check(ids, mask=mask)


def test_lookup_op_range_checks_before_device_work():
    from ultravox_b200 import ops
    z = torch.zeros(1, dtype=torch.int32)
    for k, n in ((0, 2), (32, 2), (4, 0)):
        with pytest.raises(ValueError):
            ops.lookup_draft(torch.zeros(8, dtype=torch.int64), z, z, 4, k, n, None, z, torch.zeros(k + 1, dtype=torch.int64), z,
                             z, z, z, z, z)
