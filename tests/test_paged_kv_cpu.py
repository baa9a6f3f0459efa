"""Host bookkeeping of the paged KV cache (serving.PagePool) and the scheduler rules built on it - page reservation and release,
sessions keeping their pages between turns, the submit-time and run-time capacity errors, FIFO waiting for pages - with a
stand-in engine, so no GPU is needed."""
import pytest
import torch

from ultravox_b200 import serving
from ultravox_b200.serving import PagePool, pages_for


def test_pages_for():
    assert [pages_for(n) for n in (0, 1, 63, 64, 65, 128, 129)] == [0, 1, 1, 1, 2, 2, 3]


def test_reserve_and_release_counts():
    pool = PagePool(10)
    a = pool.reserve(130)                       # 3 pages
    assert len(a) == 3 and pool.free_pages == 7
    b = pool.reserve(7 * 64)                    # exactly the rest
    assert len(b) == 7 and pool.free_pages == 0 and not set(a) & set(b)
    assert pool.reserve(1) is None and pool.free_pages == 0     # short: nothing taken
    pool.release(a)
    assert pool.free_pages == 3
    pool.release(b)
    assert pool.free_pages == 10 and sorted(pool._free) == list(range(10))


def test_session_keeps_pages_and_grows():
    pool = PagePool(16)
    sid = pool.open_session()
    p1 = pool.reserve(100 + 30, sid)            # turn 1: S = 100, max_new = 30 -> 3 pages
    assert len(p1) == 3 and pool.free_pages == 13
    pool.release(p1, sid, kv_len=100 + 12 - 1)  # 12 new tokens: 111 positions kept -> 2 pages
    s = pool.session(sid)
    assert s.kv_len == 111 and s.pages == p1[:2] and pool.free_pages == 14 and not s.busy
    p2 = pool.reserve(200 + 40, sid)            # turn 2 extends it: its first pages are the session's
    assert p2[:2] == p1[:2] and len(p2) == 4 and pool.free_pages == 12
    pool.release(p2, sid, kv_len=239)
    assert pool.session(sid).pages == p2[:4] and pool.free_pages == 12
    assert pool.session_pages() == 4
    pool.close_session(sid)
    assert pool.free_pages == 16 and pool.session_pages() == 0
    with pytest.raises(KeyError):
        pool.session(sid)


def test_close_session_returns_every_page():
    pool = PagePool(12)
    sids = [pool.open_session() for _ in range(3)]
    for i, sid in enumerate(sids):
        pool.release(pool.reserve(64 * (i + 1) + 5, sid), sid, kv_len=64 * (i + 1))
    assert pool.free_pages == 12 - (1 + 2 + 3)
    for sid in sids:
        pool.close_session(sid)
    assert pool.free_pages == 12
    busy = pool.open_session()
    pool.session(busy).busy = True
    with pytest.raises(RuntimeError):
        pool.close_session(busy)


# ------------------------------------------------------------------------------------------------ the scheduler's rules
class _StubEngine:
    """Just enough of PagedSlotDecodeEngine for the scheduler's admission logic."""

    def __init__(self, model, slots, max_len, kv_pages=None, eos_token_ids=None, pad_token_id=0, use_graph=True):
        self.slots, self.max_len = slots, max_len
        self.busy = [False] * slots
        self.pos = torch.zeros(slots, dtype=torch.int32)
        self.prefilling = None
        self.admitted = []

    def admit(self, slot, input_ids, max_new, *args, past=0, pages=None, **features):
        self.busy[slot] = True
        self.admitted.append((slot, int(input_ids.shape[1]), past, list(pages)))


def _sched(monkeypatch, slots=2, max_len=512, kv_pages=8):
    monkeypatch.setattr(serving, "PagedSlotDecodeEngine", _StubEngine)
    sched = serving.SlotScheduler(None, slots=slots, max_len=max_len, kv_pages=kv_pages)
    started = []
    monkeypatch.setattr(sched, "_started", lambda j, r: (started.append(r.rid), sched._running.__setitem__(j, r)))
    return sched, started


def ids(n):
    return dict(input_ids=torch.zeros(1, n, dtype=torch.int64))


def test_submit_errors(monkeypatch):
    sched, _ = _sched(monkeypatch, kv_pages=4)
    with pytest.raises(ValueError, match="KV pages"):
        sched.submit(ids(250), max_new_tokens=10)          # 5 pages > a pool of 4: could never run
    sched.submit(ids(250), max_new_tokens=6)               # exactly 4 pages
    with pytest.raises(ValueError, match="unknown or closed"):
        sched.submit(ids(10), max_new_tokens=2, session=123)
    sid = sched.open_session()
    sched.submit(ids(10), max_new_tokens=2, session=sid)
    with pytest.raises(ValueError, match="in flight"):
        sched.submit(ids(20), max_new_tokens=2, session=sid)
    with pytest.raises(RuntimeError, match="in flight"):
        sched.close_session(sid)
    sched.pool.session(sid).busy = False
    sched.pool.session(sid).kv_len = 30
    with pytest.raises(ValueError, match="extend"):
        sched.submit(ids(30), max_new_tokens=2, session=sid)
    sched.close_session(sid)
    with pytest.raises(ValueError, match="unknown or closed"):
        sched.session_length(sid)
    monkeypatch.setattr(serving, "SlotDecodeEngine", _StubEngine)
    plain = serving.SlotScheduler(None, slots=2, max_len=64)
    with pytest.raises(ValueError, match="kv_pages"):
        plain.open_session()
    with pytest.raises(ValueError, match="kv_pages"):
        plain.submit(ids(10), max_new_tokens=2, session=0)


def test_fifo_waits_for_pages(monkeypatch):
    sched, started = _sched(monkeypatch, slots=4, kv_pages=5)
    a = sched.submit(ids(200), max_new_tokens=20)          # 4 pages
    b = sched.submit(ids(60), max_new_tokens=10)           # 2 pages: must wait although a slot and 1 page are free
    c = sched.submit(ids(10), max_new_tokens=5)            # 1 page: would fit, but FIFO keeps it behind b
    sched._admit()
    assert started == [a] and sched.pool.free_pages == 1
    assert [r.rid for r in sched._queue] == [b, c]
    sched.pool.release(sched._running.pop(0).pages)        # a retires
    sched.engine.busy[0] = False
    sched._admit()
    assert started == [a, b, c] and sched.pool.free_pages == 5 - 2 - 1


def test_run_raises_when_sessions_hold_the_pool(monkeypatch):
    sched, _ = _sched(monkeypatch, slots=2, kv_pages=4)
    sid = sched.open_session()
    sched.pool.release(sched.pool.reserve(3 * 64, sid), sid, kv_len=3 * 64)   # the session keeps 3 pages between turns
    assert sched.free_pages == 1
    sched.submit(ids(100), max_new_tokens=10)              # 2 pages: fits the pool, not what the sessions leave free
    with pytest.raises(RuntimeError, match="open sessions hold 3"):
        sched.run()
    sched.close_session(sid)
    assert sched.free_pages == 4
