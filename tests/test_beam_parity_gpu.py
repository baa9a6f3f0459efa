"""Per-op parity of the beam-search kernels (generate.cu ``uvx_log_softmax``, ``uvx_beam_select``, ``uvx_beam_update`` /
``_stop``, ``uvx_kv_reorder``, ``uvx_stop_strings_beam``) against the host oracles of tests/test_beam_parity_cpu.py.

Bounds.
* log_softmax: per element, |y - y64| <= u|d| + E + u(|d| + |lse| + E) (x 1.01), u = 2^-24, d = x - max, E the lse error of
  ceil(V/1024) - 1 + 10 summation levels of expf terms within 2 ulp and a logf within 1 ulp (derived in
  ``test_beam_parity_cpu.log_softmax_ref``); the fraction of it used is printed.  -inf of the reference is -inf bit for
  bit.  An all-(-inf) row gives NaN, as torch.log_softmax does; the engine cannot produce one, because it runs log_softmax
  on the raw LM-head logits and applies the token constraints (the only source of -inf) afterwards.
* Everything else is exact: beam_select values (bit patterns) and flat indices, its per-row scratch, every state array of
  beam_update after every step against transformers' helpers with ties broken towards the lower index, kv_reorder on raw
  int16 views (NaN payloads included), and each stop-string hit.

Planted faults, each built once into a scratch copy of generate.cu and caught here:
1. beam_merge_kernel ties towards the higher index: test_beam_select, test_beam_update_hf.
2. radix select ``hist[d] >= rem`` -> ``>``: an equivalent mutant, caught by nothing: skipping a bucket that holds exactly
   the remaining count leaves rem = 0, so the threshold drops below the K set, no key is taken at it, and the same K keys
   lie above it.
3. inclusive rank scan in beam_row_topk_kernel: test_beam_select.
4. ``did`` without ``tid < nb``: test_beam_update_hf.
5. pool merge ties reversed (new before old): test_beam_update_hf.
6. sequence staging of the first 128-position chunk only: test_beam_update_hf (S = 120 / 250 / 127 / 255).
7. the last CTA folds only its own prompt's flags: test_beam_update_hf (B = 7, 33).
8. kv_reorder stages a parent only when ``par[c] == c + 1``: test_kv_reorder.
9. log_softmax sums exp(x) without subtracting the max: test_log_softmax."""
import math

import pytest
import torch

from test_beam_parity_cpu import HFBeams, check_log_softmax, log_softmax_rows, select_ref

pytestmark = pytest.mark.gpu

V_LLAMA = 128256


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16).cpu()


# ------------------------------------------------------------------------------------------------------------------------
# 1. log_softmax

@pytest.mark.parametrize("V", [V_LLAMA, 32000, 1024, 1000, 7, 1])
def test_log_softmax(ops, V):
    g = torch.Generator().manual_seed(V + 1)
    x = log_softmax_rows(V, g)
    got = ops.log_softmax(x.cuda()).cpu()
    frac = check_log_softmax(got, x)
    assert bool((got[3] == got[3, 0]).all())                              # a constant row: one value, -log V
    assert float(got[4, (V * 2) // 3]) == 0.0 and int(torch.isneginf(got[4]).sum()) == V - 1
    xi = x.cuda()
    ops.log_softmax(xi, out=xi)                                            # in place
    assert torch.equal(bits(xi), bits(got))
    allinf = ops.log_softmax(torch.full((1, V), -math.inf, device="cuda")).cpu()
    assert bool(torch.isnan(allinf).all())                                # as torch.log_softmax
    print(f"log_softmax V={V}: {frac:.3f} of the bound")


# ------------------------------------------------------------------------------------------------------------------------
# 2. beam_select

SELECT_NB_EOS = [(2, 0), (2, 3), (2, 7), (3, 0), (3, 3), (3, 7), (5, 0), (5, 3), (5, 7), (8, 0), (8, 3), (8, 7)]
PATTERNS = ("random", "tie_spread", "eq_K", "eq_Km1", "eq_Kp1", "zeros", "first_step", "first_step_banned", "large",
            "few_finite", "permuted")


def select_prompt(pat: str, nb: int, V: int, K: int, g: torch.Generator):
    """lp [nb, V] fp32, sc [nb] fp32 of one prompt aimed at one path of beam_row_topk_kernel / beam_merge_kernel."""
    c = -(-V // 1024)
    lp = -20.0 - 10.0 * torch.rand(nb, V, generator=g)
    sc = -torch.rand(nb, generator=g) * 5
    flat = lp.view(-1)
    if pat == "random":
        lp = torch.log_softmax(torch.randn(nb, V, generator=g) * 3, -1)
    elif pat == "tie_spread":
        # the K-th value tied over many chunks (t*c, t*c + c - 1), warps and beams; a few entries above it
        sc.fill_(-2.0)
        t = torch.arange(0, 1024, 3)
        pos = torch.cat([t * c, t * c + c - 1])
        pos = pos[pos < V]
        for j in range(nb):
            lp[j, pos] = -1.5
        above = torch.randperm(nb * V, generator=g)[:K // 2]
        flat[above] = -1.0 + torch.rand(above.numel(), generator=g) * 0.5
    elif pat in ("eq_K", "eq_Km1", "eq_Kp1"):
        m = K + {"eq_K": 0, "eq_Km1": -1, "eq_Kp1": 1}[pat]
        sc.fill_(-1.0)
        m = min(m, nb * V)
        flat[torch.randperm(nb * V, generator=g)[:m]] = -0.25
    elif pat == "zeros":
        sc.fill_(-0.0)
        lp = -1.0 - torch.rand(nb, V, generator=g)
        flat = lp.view(-1)
        n_pos = K // 3
        idx = torch.randperm(nb * V, generator=g)
        flat[idx[:n_pos]] = 0.5
        z = idx[n_pos:n_pos + 2 * K]
        flat[z] = torch.where(torch.arange(z.numel()) % 2 == 0, torch.tensor(-0.0), torch.tensor(0.0))
    elif pat in ("first_step", "first_step_banned"):
        lp = torch.log_softmax(torch.randn(nb, V, generator=g) * 3, -1)
        sc.fill_(-1e9)
        sc[0] = 0.0
        if pat == "first_step_banned":
            lp[0, torch.randperm(V, generator=g)[:V - max(1, K // 3)]] = -math.inf
    elif pat == "large":
        sc = -300.0 - torch.rand(nb, generator=g)
        lp = torch.log_softmax(torch.randn(nb, V, generator=g), -1)
    elif pat == "few_finite":
        lp = torch.full((nb, V), -math.inf)
        flat = lp.view(-1)
        keep = torch.randperm(nb * V, generator=g)[:max(1, K // 2)]
        flat[keep] = torch.randn(keep.numel(), generator=g)
        lp[:, 0] = -math.inf
        lp[:, V - 1] = -math.inf
    elif pat == "permuted":
        sc.fill_(-3.0)
        lp = -0.5 * torch.randint(0, 8, (nb, V), generator=g).float()
        lp = lp[:, torch.randperm(V, generator=g)]
    return lp.float().contiguous(), sc.float()


@pytest.mark.parametrize("V", [V_LLAMA, 32000, 1000, 0])
@pytest.mark.parametrize("nb,n_eos", SELECT_NB_EOS)
def test_beam_select(ops, nb, n_eos, V):
    """Every pattern at B = 1, 4 and 8 (V = 0: V = K); values by bit pattern, flat indices, and the per-row scratch."""
    K = max(2, 1 + n_eos) * nb
    V = V or K
    g = torch.Generator().manual_seed(1000 * nb + 10 * n_eos + V % 997)
    prompts = [select_prompt(p, nb, V, K, g) for p in PATTERNS]
    i = 0
    for B in (1, 4, 8):
        chunk = [prompts[(i + b) % len(prompts)] for b in range(B)]
        i += B
        lp = torch.cat([c[0] for c in chunk])
        sc = torch.cat([c[1] for c in chunk])
        row_s, row_i, out_s, out_i = select_ref(lp, sc, nb, K)
        scratch = (torch.full((B * nb * K,), float("nan"), device="cuda"), torch.full((B * nb * K,), -1, dtype=torch.int64,
                                                                                         device="cuda"))
        s, ix = ops.beam_select(lp.cuda(), sc.cuda(), nb, K, scratch=scratch)
        case = (nb, n_eos, V, B)
        assert torch.equal(ix.cpu(), out_i), case
        assert torch.equal(bits(s), bits(out_s)), case
        assert torch.equal(scratch[1].view(B * nb, K).cpu(), row_i), case
        assert torch.equal(bits(scratch[0].view(B * nb, K)), bits(row_s)), case


# ------------------------------------------------------------------------------------------------------------------------
# 3. beam_update / beam_update_stop against transformers' helpers

ES = {False: 0, True: 1, "never": 2}
STATE_KEYS = ("run_score", "pool_score", "pool_len", "pool_fin", "parent", "tok", "heur", "flags")


def new_state(prompt: torch.Tensor, nb: int, L: int, stride: int):
    """The engine's buffers (BeamDecodeEngine.begin) with sequences of row stride ``stride`` > L: [L, stride) holds -7."""
    B, S = prompt.shape
    R = B * nb
    dev = torch.device("cuda")
    i32 = dict(dtype=torch.int32, device=dev)
    seq = torch.zeros(R, stride, dtype=torch.int64, device=dev)
    seq[:, L:] = -7
    seq[:, :S] = prompt.repeat_interleave(nb, 0).to(dev)
    run_score = torch.full((B, nb), -1e9, device=dev)
    run_score[:, 0] = 0.0
    st = dict(run_score=run_score.view(-1), run_seq=seq, pool_seq=seq.clone(), pool_score=torch.full((R,), -1e9, device=dev),
              pool_len=torch.zeros(R, **i32), pool_fin=torch.zeros(R, **i32), parent=torch.arange(R, **i32) // nb * nb,
              tok=torch.zeros(R, dtype=torch.int64, device=dev), heur=torch.ones(B, **i32), flags=torch.zeros(B, **i32),
              ticket=torch.zeros(1, **i32))
    cnt = dict(cur_len=torch.full((1,), S, **i32), step_idx=torch.zeros(1, **i32), done=torch.zeros(1, **i32))
    bumps = tuple(torch.full((R,), 5 * k, **i32) for k in range(3))
    return st, cnt, bumps


def snapshot(st, cnt, bumps) -> dict:
    out = {k: v.cpu().clone() for k, v in st.items()}
    out.update({k: v.cpu().clone() for k, v in cnt.items()})
    out["bumps"] = torch.stack([b.cpu() for b in bumps])
    return out


def assert_same(a: dict, b: dict, case):
    for k in a:
        assert torch.equal(a[k].view(torch.int32) if a[k].dtype == torch.float32 else a[k],
                           b[k].view(torch.int32) if b[k].dtype == torch.float32 else b[k]), (case, k)


def update_logprobs(B: int, nb: int, V: int, eos: list, t: int, g: torch.Generator) -> torch.Tensor:
    """Quarter-step log-probs (sums exact, so scores tie often).  Prompt mode (b + t) % 3 / b % 4 == 3: EOS on top, EOS
    around rank nb (hits outside the top nb), EOS far down; prompts with b % 4 == 3 always finish early."""
    lp = -0.25 * torch.randint(1, 40, (B, nb, V), generator=g).float()
    if eos:
        e = torch.tensor(eos)
        for b in range(B):
            mode = 0 if b % 4 == 3 else (b + t) % 3
            lo, hi = ((0, 2), (3, 8), (30, 40))[mode]
            lp[b][:, e] = -0.25 * torch.randint(lo, hi, (nb, len(eos)), generator=g).float()
    return lp.view(B * nb, V)


def run_update_case(ops, nb, n_eos, B, lpen, es, max_new, S, V, stop, g, ev):
    K = max(2, 1 + n_eos) * nb
    eos = list(range(7, 7 + 13 * n_eos, 13))
    L = S + max_new
    stride = L + 37
    prompt = torch.randint(0, V, (B, S), generator=g)
    ref = HFBeams(prompt, nb, V, K, max_new, eos, lpen, es)
    st, cnt, bumps = new_state(prompt, nb, L, stride)
    twin = new_state(prompt, nb, L, stride) if not stop else None     # uvx_beam_update_stop with an all-zero mask
    eos_d = torch.tensor(eos, dtype=torch.int64, device="cuda") if eos else None
    len_div = torch.tensor([1.0] + [float(n) ** lpen for n in range(1, L + 2)], dtype=torch.float32, device="cuda")
    zero = torch.zeros(B * K, dtype=torch.int32, device="cuda")
    case = (nb, n_eos, B, lpen, es, max_new, S, stop)
    steps = 0
    for t in range(max_new):
        lp = update_logprobs(B, nb, V, eos, t, g)
        s, i = ops.beam_select(lp.cuda(), st["run_score"], nb, K)
        mask = None
        hit = None
        if stop:
            mask = torch.rand(B, K, generator=g) < (0.05, 0.3, 1.0)[t % 3] * (t % 4 != 3)
            hit = mask.view(-1).int().cuda()
        ops.beam_update(s, i, V, nb, eos_d, max_new, len_div, ES[es], lpen > 0, st, cnt, bumps, hit=hit)
        if twin is not None:
            ts, tc, tb = twin
            s2, i2 = ops.beam_select(lp.cuda(), ts["run_score"], nb, K)
            ops.beam_update(s2, i2, V, nb, eos_d, max_new, len_div, ES[es], lpen > 0, ts, tc, tb, hit=zero)
        info = ref.step(lp, mask)
        steps += 1
        got = snapshot(st, cnt, bumps)
        want = ref.state()
        cur = ref.cur
        for k in STATE_KEYS:
            assert torch.equal(got[k].view(torch.int32) if k in ("run_score", "pool_score") else got[k],
                               want[k].view(torch.int32) if k in ("run_score", "pool_score") else want[k]), (case, t, k)
        for k in ("run_seq", "pool_seq"):
            assert torch.equal(got[k][:, :cur], want[k][:, :cur]), (case, t, k)
            assert bool((got[k][:, L:] == -7).all()), (case, t, k, "past the row")
        assert int(got["done"]) == int(not ref.go) and int(got["cur_len"]) == cur and int(got["step_idx"]) == t + 1, (case, t)
        assert int(got["ticket"]) == 0 and torch.equal(got["bumps"], torch.stack([torch.full((B * nb,), 5 * k + t + 1,
                                                                                             dtype=torch.int32)
                                                                                  for k in range(3)])), (case, t)
        if twin is not None:
            assert_same(got, snapshot(*twin), (case, t, "stop with zero hits"))
        hits = info["hits"]
        ev["all_hit"] += int(hits.all(-1).any())
        ev["hit_outside_top_nb"] += int(hits[:, nb:].any())
        fin_b = (~ref.heur.view(-1)) | ref.fin.all(-1)
        ev["prompt_ends_early"] += int(ref.go and bool(fin_b.any()) and B > 1)
        old, new = info["old_pool"], info["cand_pool"]
        ev["pool_tie_old_new"] += int(bool(((old[:, :, None] == new[:, None, :]) & (old[:, :, None] > -1e8)).any()))
        ev["cut_tie"] += int(bool((info["cand"][0][:, nb - 1] == info["cand"][0][:, nb]).any()))
        if not ref.go:
            break
    # done already set: only parent changes, to the identity
    before = snapshot(st, cnt, bumps)
    lp = update_logprobs(B, nb, V, eos, max_new, g)
    s, i = ops.beam_select(lp.cuda(), st["run_score"], nb, K)
    if int(cnt["done"]):
        ops.beam_update(s, i, V, nb, eos_d, max_new, len_div, ES[es], lpen > 0, st, cnt, bumps,
                        hit=torch.ones(B * K, dtype=torch.int32, device="cuda") if stop else None)
        after = snapshot(st, cnt, bumps)
        assert torch.equal(after["parent"], torch.arange(B * nb, dtype=torch.int32)), case
        after["parent"] = before["parent"]
        assert_same(after, before, (case, "done"))
        ev["done_call"] += 1
    return steps


@pytest.mark.parametrize("stop", [False, True])
@pytest.mark.parametrize("nb", [2, 5, 8])
def test_beam_update_hf(ops, nb, stop):
    """B in (1, 7, 33) x length_penalty x early_stopping x max_new, n_eos rotating so K reaches 64 at nb = 8; prompts of
    120 / 250 (127 / 255 at max_new 1 / 2) positions, so cur_len crosses 128 and 256."""
    g = torch.Generator().manual_seed(nb * 2 + stop)
    V = 1000
    ev = dict(all_hit=0, hit_outside_top_nb=0, prompt_ends_early=0, pool_tie_old_new=0, cut_tie=0, done_call=0)
    steps = cases = 0
    for li, lpen in enumerate((1.0, 0.0, -0.5, 2.0)):
        n_eos = (0, 1, 3, 7)[li] if nb != 8 else (7, 1, 3, 7)[li]
        for es in (False, True, "never"):
            for B in (1, 7, 33):
                for max_new in (1, 2, 20):
                    S = {1: 127, 2: 255}.get(max_new, (120, 250)[(li + B) % 2])
                    steps += run_update_case(ops, nb, n_eos, B, lpen, es, max_new, S, V, stop, g, ev)
                    cases += 1
    print(f"beam_update nb={nb} stop={stop}: {cases} cases, {steps} steps, events {ev}")
    for k, n in ev.items():
        assert n >= 1, (k, ev)


# ------------------------------------------------------------------------------------------------------------------------
# 4. kv_reorder

def reorder_maps(B: int, nb: int) -> list:
    base = [list(range(nb)), [0] * nb, [1, 0] + list(range(2, nb)),
            ([1, 2, 0] + list(range(3, nb))) if nb >= 3 else [1, 0], [(j + 1) % nb for j in range(nb)],
            [nb - 1 - j if j % 2 else j // 2 for j in range(nb)]]
    out = [[b * nb + m[j] for b in range(B) for j in range(nb)] for m in base]
    # several prompts, each with a different map; prompt 1 keeps the identity (its rows are a sentinel)
    out.append([b * nb + (base[(b * 2 + 1) % len(base)] if b != 1 else base[0])[j] for b in range(B) for j in range(nb)])
    return out


def reorder_case(ops, L, B, nb, hkv, d, n_pos, smax, maps, g):
    shape = (L, B * nb, smax, hkv, d)
    k0 = torch.randint(-32768, 32768, shape, dtype=torch.int32, device="cuda", generator=g).to(torch.int16)
    v0 = torch.randint(-32768, 32768, shape, dtype=torch.int32, device="cuda", generator=g).to(torch.int16)
    n = torch.tensor([n_pos], dtype=torch.int32, device="cuda")
    for par in maps:
        p = torch.tensor(par, dtype=torch.int32, device="cuda")
        k, v = k0.clone(), v0.clone()
        ops.kv_reorder_(k.view(torch.bfloat16), v.view(torch.bfloat16), p, n, nb)
        ek, ev = k0.clone(), v0.clone()
        ek[:, :, :n_pos] = k0[:, :, :n_pos].index_select(1, p.long())
        ev[:, :, :n_pos] = v0[:, :, :n_pos].index_select(1, p.long())
        assert torch.equal(k, ek) and torch.equal(v, ev), (hkv * d, nb, n_pos, par)


@pytest.mark.parametrize("nb", [2, 3, 8])
@pytest.mark.parametrize("hkv,d", [(1, 128), (8, 64), (8, 128)])
def test_kv_reorder(ops, hkv, d, nb):
    """row_elems 128 / 512 / 1024; n_pos at P - 1, P, P + 1 and 5P + P/2 + 3 (P = 32768 / (nb * 4 * row_elems), in [1, 64])."""
    g = torch.Generator(device="cuda").manual_seed(hkv * d + nb)
    P = max(1, min(64, 32768 // (nb * 4 * hkv * d)))
    B = 3
    maps = reorder_maps(B, nb)
    for n_pos in sorted({max(1, P - 1), P, P + 1, 5 * P + P // 2 + 3}):
        reorder_case(ops, 2, B, nb, hkv, d, n_pos, n_pos + 9, maps, g)


def test_kv_reorder_begin_broadcast(ops):
    """begin(): parent = b * nb at a 4000-position prompt, 8B widths, nb = 8."""
    g = torch.Generator(device="cuda").manual_seed(4000)
    B, nb = 2, 8
    reorder_case(ops, 2, B, nb, 8, 128, 4000, 4011, [[r // nb * nb for r in range(B * nb)]], g)


# ------------------------------------------------------------------------------------------------------------------------
# 5. stop_strings_beam

def test_stop_strings_beam(ops):
    """K = 64, B 1..8, cur_len 0..300: each candidate's hit equals uvx_stop_strings on its explicit sequence (parent's
    running sequence + token) and the numpy walk."""
    from test_stop_strings_cpu import make_tokenizer
    from ultravox_b200 import stop_strings as ss
    V, nb, K = 1024, 8, 64
    tok = make_tokenizer(V, "bytelevel", seed=5)
    st = ss.StopStrings.build(tok, ["user:", "ab", "ne.", "\nx"])
    tab = st.device_table("cuda")
    text = tok(" the user: hello ab there, done.\nxyz user: ok ab ne. ab", add_special_tokens=False)["input_ids"]
    pool = torch.tensor(text)
    rng = torch.Generator().manual_seed(7)
    hits = total = 0
    for B in (1, 3, 8):
        for cur in (0, 1, 2, 5, 31, 32, 33, 128, 255, 300):
            W = cur + 5
            run_seq = torch.randint(0, V, (B * nb, W), generator=rng)
            src = pool[torch.randint(0, pool.numel(), (B * nb, W), generator=rng)]
            run_seq = torch.where(torch.rand(B * nb, W, generator=rng) < 0.7, src, run_seq)
            run_seq[:, cur:] = -1                                           # never read
            parent = torch.randint(0, nb, (B, K), generator=rng)
            tk = torch.where(torch.rand(B, K, generator=rng) < 0.8, pool[torch.randint(0, pool.numel(), (B, K), generator=rng)],
                             torch.randint(0, V, (B, K), generator=rng))
            cand_i = (parent * V + tk).contiguous()
            cl = torch.tensor([cur], dtype=torch.int32, device="cuda")
            hit = torch.full((B * K,), -5, dtype=torch.int32, device="cuda")
            ops.stop_strings_beam(cand_i.cuda(), V, nb, run_seq.cuda(), cl, tab, hit)
            rows = (torch.arange(B)[:, None] * nb + parent).view(-1)
            seqs = run_seq[rows].contiguous()
            plain = torch.full((B * K,), -5, dtype=torch.int32, device="cuda")
            ops.stop_strings(tk.view(-1).cuda(), seqs.cuda(), cl, tab, plain)
            walk = torch.tensor([int(ss.walk(st.table, seqs[r, :cur].tolist() + [int(tk.view(-1)[r])])) for r in range(B * K)],
                                dtype=torch.int32)
            assert torch.equal(hit.cpu(), walk), (B, cur)
            assert torch.equal(plain.cpu(), walk), (B, cur)
            hits += int(walk.sum())
            total += walk.numel()
    print(f"stop_strings_beam: {hits} hits of {total}")
    assert 0 < hits < total
