"""Host swap of idle sessions, host side: serving.PagePool's host tier (the invariants of both tiers under random operations,
the swap-out policy: LRU order, busy sessions and the waiting request's own never picked, all-or-nothing on the freed pages
and on host room), the scheduler's admission with a stand-in engine that tracks what each page holds (so a swapped-in
session finds its own contents), its error message and argument checks, and the new entry point's ABI binding."""
import ctypes
import random

import pytest
import torch

from ultravox_b200 import _lib, serving
from ultravox_b200.serving import PAGE, PagePool

from test_prefix_cache_cpu import check, toks


def check_tiers(pool: PagePool, running=()):
    """Both tiers' invariants: every device page free, reclaimable or held with the right count (``check``); every host
    page free or held by exactly one session; each session on exactly one side; counts conserved."""
    sessions = pool._sessions.values()
    check(pool, [s.pages for s in sessions] + list(running))
    host_held = [p for s in sessions for p in s.host]
    assert len(host_held) == len(set(host_held)) and not set(host_held) & set(pool._host_free)
    assert len(pool._host_free) == len(set(pool._host_free))
    assert sorted(host_held + pool._host_free) == list(range(pool.host_pages))
    for s in sessions:
        assert not (s.host and s.pages)
        if s.host:
            assert len(s.host) == serving.pages_for(s.kv_len) and not s.busy


def keep_session(pool, sid, positions):
    """A session that has run one turn and keeps ``positions`` positions."""
    pool.release(pool.reserve(positions + 10, sid), sid, positions)


# ------------------------------------------------------------------------------------------------ PagePool
def test_random_operations_keep_both_tiers_consistent():
    rng = random.Random(4321)
    pool = PagePool(24, host_pages=10)
    prompts = [toks(200 + k, 3) for k in range(3)]
    running, busy = [], set()                           # running: [pages, sid or None, prefix, registered]
    sessions = []
    for step in range(4000):
        op = rng.choice(["admit", "admit", "register", "retire", "open", "close", "swap", "swap", "policy"])
        idle = [s for s in sessions if s not in busy]
        if op == "open" and len(sessions) < 6:
            sessions.append(pool.open_session())
        elif op == "close" and idle:
            sid = rng.choice(idle)
            pool.close_session(sid)
            sessions.remove(sid)
        elif op == "swap" and idle:
            sid = rng.choice(idle)
            s = pool.session(sid)
            if len(s.pages) > pool.host_free_pages:
                with pytest.raises(ValueError, match="host tier"):
                    pool.swap_out(sid)
            else:
                before = list(s.pages)
                dev, host = pool.swap_out(sid)
                assert dev == before and len(host) == len(dev)
        elif op == "policy":
            need = rng.randint(1, 8)
            excl = rng.choice(sessions + [None])
            got = pool.swap_candidates(need, excl)
            if got is not None:
                assert excl not in got and not set(got) & busy
                for sid in got:
                    pool.swap_out(sid)
        elif op == "admit":
            pt = rng.choice(prompts)[:rng.randint(0, 3)]
            positions = len(pt) * PAGE + rng.randint(1, 150)
            sid = rng.choice(idle + [None, None])
            shared = []
            if sid is not None and pool.session(sid).kv_len:
                pt = ()
                positions = pool.session(sid).kv_len + rng.randint(1, 100)
            else:
                shared = pool.match(pt[:(positions - 1) // PAGE])
            host = list(pool.session(sid).host) if sid is not None else []
            free_host = pool.host_free_pages
            short = pool.shortfall(positions, sid, shared)
            pages = pool.reserve(positions, sid, shared)
            assert (pages is None) == (short > 0)
            if pages is None:
                check_tiers(pool, [r[0] for r in running if r[1] is None])
                continue
            assert pool.host_free_pages == free_host + len(host)
            if host:
                assert not set(pages) & {p for r in running for p in r[0]}                  # restored pages are private
            running.append([pages, sid, pt, False])
            if sid is not None:
                busy.add(sid)
                pool.session(sid).busy = True
        elif op == "register" and running:
            r = rng.choice(running)
            if not r[3] and r[2]:
                pool.register(r[0], r[2])
                r[3] = True
        elif op == "retire" and running:
            pages, sid, _, _ = running.pop(rng.randrange(len(running)))
            if sid is None:
                pool.release(pages)
            else:
                pool.release(pages, sid, rng.randint(len(pages) * PAGE - 63, len(pages) * PAGE) - 1)
                busy.discard(sid)
        check_tiers(pool, [r[0] for r in running if r[1] is None])
    for pages, sid, _, _ in running:
        pool.release(pages, sid, 0) if sid is not None else pool.release(pages)
    for sid in sessions:
        pool.close_session(sid)
    check_tiers(pool)
    assert pool.free_pages == 24 and pool.host_free_pages == 10


def test_policy_takes_least_recently_used_first():
    pool = PagePool(12, host_pages=12)
    a, b, c = (pool.open_session() for _ in range(3))
    keep_session(pool, b, 2 * PAGE)                     # b retires first, then c, then a
    keep_session(pool, c, 2 * PAGE)
    keep_session(pool, a, 2 * PAGE)
    assert pool.swap_candidates(1) == [b]
    assert pool.swap_candidates(2) == [b]
    assert pool.swap_candidates(3) == [b, c]
    assert pool.swap_candidates(6) == [b, c, a]
    assert pool.swap_candidates(7) is None              # all of them free only 6 pages
    assert pool.swap_candidates(3, exclude=b) == [c, a]
    pool.session(c).busy = True                         # a turn of c is queued: c stays
    assert pool.swap_candidates(3) == [b, a]
    keep_session(pool, c, 2 * PAGE)                     # retiring again makes c the most recent
    assert pool.swap_candidates(6) == [b, a, c]
    check_tiers(pool)


def test_policy_counts_only_pages_a_swap_frees():
    pool = PagePool(16, host_pages=16)
    pre = toks(9, 2)
    donor = pool.reserve(2 * PAGE + 5)
    pool.register(donor, pre)
    a, b = pool.open_session(), pool.open_session()
    for sid in (a, b):                                  # both share the 2 cached pages and add 1 private page each
        pool.release(pool.reserve(3 * PAGE, sid, shared=pool.match(pre)), sid, 3 * PAGE - 1)
    assert pool.session(a).pages[:2] == pool.session(b).pages[:2] == donor[:2]
    assert pool.swap_candidates(1) == [a]               # a's private page
    assert pool.swap_candidates(2) == [a, b]            # b's private page; the shared ones are still held by the donor
    assert pool.swap_candidates(3) is None
    pool.release(donor)                                 # now only the sessions hold the shared pages
    assert pool.swap_candidates(3) == [a, b]            # both swapped: the 2 shared pages become reclaimable too
    assert pool.swap_candidates(4) == [a, b]
    assert pool.swap_candidates(5) is None
    # pages the waiting request takes from the cache itself do not count as freed for it
    assert pool.swap_candidates(3, keep=donor[:2]) is None
    assert pool.swap_candidates(2, keep=donor[:2]) == [a, b]
    dev, host = pool.swap_out(a)
    assert dev == pool.session(b).pages[:2] + dev[2:] and pool._refs[donor[0]] == 1
    dev, host = pool.swap_out(b)
    assert pool.free_pages == 16 and len(pool._reclaimable) == 2 and pool.match(pre) == donor[:2]
    check_tiers(pool)


def test_policy_respects_host_room():
    pool = PagePool(10, host_pages=3)
    a, b = pool.open_session(), pool.open_session()
    keep_session(pool, a, 2 * PAGE)
    keep_session(pool, b, 2 * PAGE)
    assert pool.swap_candidates(2) == [a]
    assert pool.swap_candidates(3) is None              # a and b need 4 host pages, the tier has 3
    pool.swap_out(a)
    assert pool.host_free_pages == 1
    assert pool.swap_candidates(1) is None              # b alone needs 2
    with pytest.raises(ValueError, match="host tier has 1 free"):
        pool.swap_out(b)
    assert pool.swap_out(a) == ([], [])                 # already on the host: nothing to move
    check_tiers(pool)
    pool.close_session(a)
    assert pool.host_free_pages == 3
    check_tiers(pool)


def test_swap_in_by_reservation():
    pool = PagePool(8, host_pages=4)
    sid = pool.open_session()
    keep_session(pool, sid, 2 * PAGE + 3)               # 3 pages
    dev, host = pool.swap_out(sid)
    assert len(dev) == 3 and pool.free_pages == 8 and pool.session(sid).pages == [] and pool.session(sid).host == host
    with pytest.raises(ValueError, match="in flight"):
        pool.session(sid).busy = True
        pool.swap_out(sid)
    other = pool.reserve(4 * PAGE)                      # leaves 4 device pages
    assert pool.reserve(5 * PAGE, sid) is None and pool.session(sid).host == host      # waits, stays on the host
    assert pool.shortfall(5 * PAGE, sid) == 1
    got = pool.reserve(4 * PAGE, sid)
    assert len(got) == 4 and not set(got) & set(other)
    assert pool.session(sid).pages == got and pool.session(sid).host == [] and pool.host_free_pages == 4
    pool.release(got, sid, 3 * PAGE)
    pool.release(other)
    check_tiers(pool)


def test_pool_argument_checks():
    with pytest.raises(ValueError, match="host tier"):
        PagePool(4, host_pages=-1)
    assert PagePool(4).host_pages == 0 and PagePool(4).host_free_pages == 0


# ------------------------------------------------------------------------------------------------ the scheduler
class _StubEngine:
    """Admission and page moves without a GPU: ``content[page]`` is what a device page holds, ``host[page]`` a host page."""

    def __init__(self, model, slots, max_len, kv_pages=None, eos_token_ids=None, pad_token_id=0, use_graph=True,
                 host_kv_pages=0):
        self.slots, self.max_len = slots, max_len
        self.busy = [False] * slots
        self.pos = torch.zeros(slots, dtype=torch.int32)
        self.prefilling = None
        self.content, self.host = {}, {}
        self.host_kv_pages = host_kv_pages
        self.moves = []

    def admit(self, slot, input_ids, max_new, *args, past=0, pages=None, **features):
        self.busy[slot] = True
        for k in range(serving.pages_for(past)):       # the pages of the positions it keeps must hold its own K / V
            assert self.content[pages[k]] == (int(input_ids[0, 0]), k), (slot, k)
        for k in range(past // PAGE, len(pages)):      # the prefill writes [past, S)
            self.content[pages[k]] = (int(input_ids[0, 0]), k)

    def swap_out(self, dev, host):
        assert len(dev) == len(host) and all(0 <= p < self.host_kv_pages for p in host)
        self.moves.append(("out", list(dev), list(host)))
        for d, h in zip(dev, host):
            self.host[h] = self.content[d]

    def swap_in(self, host, dev):
        self.moves.append(("in", list(host), list(dev)))
        for h, d in zip(host, dev):
            self.content[d] = self.host.pop(h)


def _sched(monkeypatch, slots=2, kv_pages=8, host_kv_pages=8):
    monkeypatch.setattr(serving, "PagedSlotDecodeEngine", _StubEngine)
    sched = serving.SlotScheduler(None, slots=slots, max_len=1024, kv_pages=kv_pages, host_kv_pages=host_kv_pages)
    monkeypatch.setattr(sched, "_started", lambda j, r: sched._running.__setitem__(j, r))
    return sched


def _retire_all(sched):
    for j, r in list(sched._running.items()):
        sched.pool.release(r.pages, r.session, int(r.input_ids.shape[1]) - 1)
        sched.engine.busy[j] = False
    sched._running.clear()


def _turn(sched, sid, first_id, S, n=4):
    """A turn of ``S`` prompt tokens whose first token names the conversation."""
    ids = torch.full((1, S), 7, dtype=torch.int64)
    ids[0, 0] = first_id
    return sched.submit(dict(input_ids=ids), max_new_tokens=n, session=sid)


def test_scheduler_swaps_lru_idle_sessions_and_restores_them(monkeypatch):
    sched = _sched(monkeypatch)
    a, b, c = (sched.open_session() for _ in range(3))
    for sid, first in ((a, 100), (b, 200)):              # a and b keep 3 pages each: 2 of 8 stay free
        _turn(sched, sid, first, 2 * PAGE + 40)
        sched._admit()
        _retire_all(sched)
    assert sched.free_pages == 2 and not sched.session_on_host(a)
    _turn(sched, c, 300, 3 * PAGE)                       # needs 4: swaps out a (least recent), which frees 3
    sched._admit()
    assert sched.session_on_host(a) and not sched.session_on_host(b) and sched.swapped_out_pages == 3
    assert sched.host_free_pages == 5 and sched.free_pages == 1
    _retire_all(sched)                                   # c keeps 3 pages: 2 free
    _turn(sched, a, 100, 2 * PAGE + 41 + 20)             # a's next turn: needs 4 device pages, restores 3 of them
    sched._admit()
    assert sched.session_on_host(b) and not sched.session_on_host(a)     # b was the least recently used idle session
    assert sched.swapped_in_pages == 3 and sched.swapped_out_pages == 6
    assert [m[0] for m in sched.engine.moves] == ["out", "out", "in"]
    r = next(iter(sched._running.values()))
    assert sched.engine.moves[-1][2] == r.pages[:3] and r.past == 2 * PAGE + 39
    _retire_all(sched)
    for sid in (a, b, c):
        sched.close_session(sid)
    assert sched.free_pages == 8 and sched.host_free_pages == 8


def test_scheduler_waits_without_moving_when_a_swap_would_not_admit(monkeypatch):
    sched = _sched(monkeypatch, slots=2, kv_pages=8, host_kv_pages=2)
    a = sched.open_session()
    _turn(sched, a, 100, 2 * PAGE + 40)
    sched._admit()
    _retire_all(sched)                                   # a holds 3 pages; the host tier has only 2
    other = sched.submit(dict(input_ids=torch.full((1, 4 * PAGE), 5, dtype=torch.int64)), max_new_tokens=128)    # 6 pages
    sched._admit()
    assert other in sched.pending() and not sched._running and sched.engine.moves == []
    with pytest.raises(RuntimeError, match="open sessions hold 3 and the host tier has 2 of 2 pages free; close some"):
        sched.run()
    assert sched.swapped_out_pages == 0


def test_offload_session(monkeypatch):
    sched = _sched(monkeypatch)
    a = sched.open_session()
    sched.offload_session(a)                             # nothing held yet: nothing to move
    assert not sched.session_on_host(a) and sched.engine.moves == []
    _turn(sched, a, 100, PAGE + 10)
    with pytest.raises(ValueError, match="in flight"):
        sched.offload_session(a)
    sched._admit()
    _retire_all(sched)
    sched.offload_session(a)
    assert sched.session_on_host(a) and sched.swapped_out_pages == 2 and sched.free_pages == 8
    sched.offload_session(a)                             # already there: a no-op
    assert sched.swapped_out_pages == 2
    assert sched.session_length(a) == PAGE + 9
    with pytest.raises(ValueError, match="unknown"):
        sched.offload_session(99)
    sched.close_session(a)
    assert sched.host_free_pages == 8


def test_offload_needs_host_room_and_a_tier(monkeypatch):
    sched = _sched(monkeypatch, host_kv_pages=1)
    a = sched.open_session()
    _turn(sched, a, 100, PAGE + 10)
    sched._admit()
    _retire_all(sched)
    with pytest.raises(ValueError, match="host tier has 1 free"):
        sched.offload_session(a)
    assert not sched.session_on_host(a)
    plain = _sched(monkeypatch, host_kv_pages=0)
    b = plain.open_session()
    with pytest.raises(ValueError, match="needs a host tier"):
        plain.offload_session(b)


def test_run_error_without_a_host_tier_is_unchanged(monkeypatch):
    sched = _sched(monkeypatch, kv_pages=6, host_kv_pages=0)
    sid = sched.open_session()
    sched.pool.release(sched.pool.reserve(4 * PAGE, sid), sid, kv_len=4 * PAGE)
    sched.submit(dict(input_ids=torch.ones(1, 199, dtype=torch.int64)), max_new_tokens=100)
    with pytest.raises(RuntimeError) as e:
        sched.run()
    assert str(e.value) == "request 0 needs 5 KV pages but only 2 of 6 are free: open sessions hold 4; close some"


def _fake_model(layers=3):
    import types
    return types.SimpleNamespace(config=types.SimpleNamespace(text_config=types.SimpleNamespace(num_hidden_layers=layers)))


@pytest.mark.parametrize("kw,msg", [
    (dict(host_kv_pages=4), "kv_pages"),
    (dict(kv_pages=8, host_kv_pages=-1), ">= 0"),
    (dict(host_kv_pages=-1), ">= 0"),
    (dict(kv_pages=8, host_kv_pages=2.5), "integer"),
    (dict(kv_pages=8, host_kv_pages=True), "integer"),
])
def test_scheduler_rejects_bad_host_tier_settings(kw, msg):
    with pytest.raises(ValueError, match=msg):
        serving.SlotScheduler(_fake_model(), slots=2, max_len=128, **kw)


# ------------------------------------------------------------------------------------------------ the C ABI
def test_kv_pages_move_is_declared_and_bound():
    sig = _lib.SIGNATURES["uvx_kv_pages_move"]
    c_i64, c_vp = ctypes.c_int64, ctypes.c_void_p
    assert sig == (ctypes.c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp])
    if not _lib.LIB_PATH.exists():
        pytest.skip("libuvx.so not built")
    assert hasattr(ctypes.CDLL(str(_lib.LIB_PATH)), "uvx_kv_pages_move")
