"""Host oracles of the beam-search parity suite (tests/test_beam_parity_gpu.py), pinned on the CPU.

* ``log_softmax_ref``: fp64 log_softmax of fp32 rows and the per-element bound of ``log_softmax_kernel``'s fp32 arithmetic
  (derivation in the GPU module's docstring); it must hold on a numpy fp32 emulation of the kernel's order of operations.
* ``topk_exact`` / ``select_ref``: the top K by (value desc, index asc), which is ``uvx_beam_select``'s documented order;
  equal to ``torch.topk`` wherever the cut has no tie.
* ``HFBeams``: one prompt batch stepped through transformers' own ``_beam_search`` helpers with ``torch.topk`` made stable
  (ties go to the lower index, as the kernels break them), so every step is defined even when scores tie.  It must reproduce
  ``GenerationMixin._beam_search`` on a tiny CPU ``LlamaForCausalLM``."""
import contextlib
import math

import numpy as np
import pytest
import torch

U = 2.0 ** -24      # unit roundoff of fp32
THREADS = 1024      # log_softmax_kernel / beam_row_topk_kernel block size


# ------------------------------------------------------------------------------------------------------------------------
# log_softmax: fp64 reference and the kernel's error bound

def log_softmax_ref(x: torch.Tensor):
    """x [R, V] fp32 -> (fp64 log_softmax [R, V], per-element bound [R, V]) for log_softmax_kernel.

    The kernel computes y = fl(fl(x - mx) - fl(log(S))), S = fl-sum of fl(expf(fl(x - mx))) with each of the 1024 threads
    summing its ceil(V / 1024) strided terms in order and then two 32-wide shuffle trees (depth 10).  With u = 2^-24:
    d~ = d (1 + a), |a| <= u; expf within 2 ulp, so e~ = e^d (1 + b), |b| <= 4u + u|d| (+ the argument error); the sum of
    n = ceil(V/1024) - 1 + 10 levels of positive terms gives |S~ - S| <= (sum e_i |b_i|)(1 + g) + g S, g = n u / (1 - n u);
    logf within 1 ulp: |lse~ - lse| <= r (1 + r) + 2u|lse|, r = |S~ - S| / S; the final subtraction rounds once more.  So
    |y~ - y| <= u|d| + E + u(|d| + |lse| + E), E = the lse error above, widened by 1 % and a 1e-37 V absolute floor for
    flushed terms."""
    x64 = x.double()
    mx = x64.max(-1, keepdim=True).values
    d = x64 - mx
    e = torch.exp(d)
    s = e.sum(-1, keepdim=True)
    lse = torch.log(s)
    y = d - lse
    V = x.shape[-1]
    n = -(-V // THREADS) - 1 + 10
    g = n * U / (1 - n * U)
    fin = torch.isfinite(d)
    dabs = torch.where(fin, d.abs(), torch.zeros_like(d))
    r = ((e * (4 * U + U * dabs)).sum(-1, keepdim=True) * (1 + g) + g * s) / s
    E = r * (1 + r) + 2 * U * lse.abs()
    bound = 1.01 * (U * dabs + E + U * (dabs + lse.abs() + E)) + 1e-37 * V
    return y, bound


def emulate_log_softmax(x: torch.Tensor) -> torch.Tensor:
    """numpy fp32 in log_softmax_kernel's order: strided per-thread sums, then 32 x 32 butterfly trees."""
    xs = x.numpy().astype(np.float32)
    R, V = xs.shape
    out = np.empty_like(xs)
    with np.errstate(over="ignore", invalid="ignore"):
        for r in range(R):
            row = xs[r]
            mx = row.max()
            part = np.zeros(THREADS, dtype=np.float32)
            for i0 in range(0, V, THREADS):
                seg = row[i0:i0 + THREADS]
                part[:seg.size] = part[:seg.size] + np.exp(seg - mx).astype(np.float32)
            for w in (32, 1):                       # lanes within warps, then across the 32 warp results
                p = part.reshape(-1, 32) if w == 32 else part.reshape(1, 32)
                p = p.copy()
                for o in (16, 8, 4, 2, 1):
                    p = p + p[:, np.arange(32) ^ o]
                part = p[:, 0].astype(np.float32)
            lse = np.float32(np.log(part[0]))
            out[r] = (row - mx).astype(np.float32) - lse
    return torch.from_numpy(out)


def log_softmax_rows(V: int, g: torch.Generator) -> torch.Tensor:
    """Rows at scale 1, 30 and 1e4, a constant row, a one-finite row and -inf at chunk ends / 0 / V - 1 (fp32 [7, V])."""
    rows = [torch.randn(V, generator=g), torch.randn(V, generator=g) * 30, torch.randn(V, generator=g) * 1e4,
            torch.full((V,), 0.375)]
    one = torch.full((V,), -math.inf)
    one[(V * 2) // 3] = 1.5
    rows.append(one)
    banned = torch.randn(V, generator=g) * 3
    c = -(-V // THREADS)
    t = torch.arange(0, THREADS, 7)                         # every 7th thread's chunk ends (a row stays mostly finite)
    ends = torch.cat([t * c + c - 1, t * c, torch.tensor([0, V - 1])])
    banned[ends[ends < V]] = -math.inf
    banned[V // 2] = 0.5
    rows.append(banned)
    lead = torch.randn(V, generator=g) * 3
    lead[:max(1, V // 2)] = -math.inf
    lead[V - 1] = 2.0
    rows.append(lead)
    return torch.stack(rows).float()


def check_log_softmax(got: torch.Tensor, x: torch.Tensor) -> float:
    """Asserts got (fp32) within the bound of log_softmax_ref(x); -inf of the reference must be -inf.  -> max fraction."""
    y, bound = log_softmax_ref(x)
    ninf = torch.isneginf(y)
    assert torch.equal(torch.isneginf(got), ninf), "-inf pattern differs"
    fin = ~ninf
    assert bool(torch.isfinite(got[fin]).all()), "non-finite output where the reference is finite"
    err = (got.double() - y).abs()[fin]
    frac = (err / bound[fin]).max().item() if err.numel() else 0.0
    assert frac <= 1.0, f"log_softmax error {frac:.3f} x bound"
    return frac


# ------------------------------------------------------------------------------------------------------------------------
# exact top K by (value desc, index asc)

def topk_exact(a: torch.Tensor, K: int):
    """a [R, N] fp32 (no NaN) -> (values [R, K], indices [R, K] int64) ordered by (value desc, index asc); -0.0 == +0.0."""
    vals, idxs = [], []
    for row in a:
        thr = torch.topk(row, K).values[-1]
        cand = torch.nonzero(row >= thr).view(-1)               # ascending index
        order = torch.sort(row[cand], descending=True, stable=True).indices[:K]
        idxs.append(cand[order])
        vals.append(row[cand[order]])
    return torch.stack(vals), torch.stack(idxs)


def select_ref(lp: torch.Tensor, sc: torch.Tensor, nb: int, K: int):
    """uvx_beam_select on the host: lp [B*nb, V] fp32 + sc [B*nb] fp32 (one fp32 add, as HF forms it) ->
    (row_s [B*nb, K], row_i [B*nb, K] = j * V + v, out_s [B, K], out_i [B, K] flat index)."""
    R, V = lp.shape
    a = lp + sc[:, None]
    row_s, row_v = topk_exact(a, K)
    row_i = row_v + (torch.arange(R) % nb)[:, None] * V
    out_s, out_i = topk_exact(a.view(R // nb, nb * V), K)
    return row_s, row_i, out_s, out_i


# ------------------------------------------------------------------------------------------------------------------------
# transformers' _beam_search helpers, step by step

@contextlib.contextmanager
def stable_topk():
    """torch.topk with ties in index order (a stable descending sort): the kernels' rule, and one valid torch.topk order."""
    orig = torch.topk

    def topk(x, k, dim=-1, largest=True, sorted=True):
        assert largest and dim in (-1, x.dim() - 1)
        s = torch.sort(x, dim=-1, descending=True, stable=True)
        return torch.return_types.topk((s.values[..., :k], s.indices[..., :k]))

    torch.topk = topk
    try:
        yield
    finally:
        torch.topk = orig


class HFBeams:
    """HF's beam state for B prompts [B, S] (pad 0 past the prompt), advanced by ``step`` through GenerationMixin's helpers."""

    def __init__(self, prompt: torch.Tensor, nb: int, V: int, K: int, max_new: int, eos, lpen: float, es):
        B, S = prompt.shape
        self.B, self.S, self.nb, self.V, self.K, self.max_new = B, S, nb, V, K, max_new
        self.L = S + max_new
        self.eos = torch.as_tensor(list(eos), dtype=torch.int64)
        self.lpen, self.es = lpen, es
        self.r_seq = torch.zeros(B, nb, self.L, dtype=torch.int64)
        self.r_seq[:, :, :S] = prompt[:, None]
        self.seqs = self.r_seq.clone()
        self.r_sc = torch.zeros(B, nb)
        self.r_sc[:, 1:] = -1e9
        self.b_sc = torch.full((B, nb), -1e9)
        self.fin = torch.zeros(B, nb, dtype=torch.bool)
        self.heur = torch.ones(B, 1, dtype=torch.bool)
        self.r_bi = torch.full((B, nb, max_new), -1, dtype=torch.int32)
        self.b_bi = self.r_bi.clone()
        self.mask = torch.cat([torch.ones(nb, dtype=torch.bool), torch.zeros(K - nb, dtype=torch.bool)])
        self.cur = S
        self.go = True
        self.parent = torch.arange(B * nb, dtype=torch.int32)
        self.tok = torch.zeros(B * nb, dtype=torch.int64)
        self.flags = torch.zeros(B, dtype=torch.int32)

    def step(self, lp: torch.Tensor, extra_hits=None) -> dict:
        """lp [B*nb, V] fp32 processed log-probs; extra_hits [B, K] bool (stop strings) -> what happened this step."""
        from transformers import GenerationMixin as G
        B, nb, V, K, S, cur = self.B, self.nb, self.V, self.K, self.S, self.cur
        with stable_topk():
            acc = (lp.view(B, nb, V) + self.r_sc[:, :, None]).view(B, nb * V)
            tlp, tseq, tbi = G._get_top_k_continuations(G, acc, self.r_seq, self.r_bi, cur, S, False, K, nb, V, B)
            hits = torch.isin(tseq[:, :, cur], self.eos) | (cur + 1 >= self.L)
            if extra_hits is not None:
                hits = hits | extra_hits
            old_b_sc = self.b_sc.clone()
            # the candidates' pool scores as _update_finished_beams forms them (for the tie events of the caller)
            cand_p = tlp / ((cur + 1 - S) ** self.lpen)
            cand_p = cand_p + (self.fin.all(-1, keepdim=True) & (self.es is True)).float() * -1.0e9
            cand_p = cand_p + (~self.heur).float() * -1.0e9
            cand_p = cand_p + (~(hits & self.mask[None])) * -1.0e9
            self.r_seq, self.r_sc, self.r_bi = G._get_running_beams_for_next_iteration(G, tlp, tseq, tbi, hits, nb)
            self.seqs, self.b_sc, self.b_bi, self.fin = G._update_finished_beams(
                G, self.seqs, tseq, self.b_sc, tlp, self.b_bi, tbi, self.heur, self.fin, hits, self.mask, nb, cur, S, self.lpen,
                self.es)
            self.heur = G._check_early_stop_heuristic(self.heur, self.r_sc, self.b_sc, self.fin, cur + 1, self.L, S, self.es,
                                                      self.lpen)
            self.go = bool(G._beam_search_has_unfinished_sequences(self.heur, self.fin, hits, self.es))
        self.parent = self.r_bi[:, :, cur - S].reshape(-1).clone()
        self.tok = self.r_seq[:, :, cur].reshape(-1).clone()
        self.flags = (self.heur.view(-1).int() | (self.fin.all(-1).int() << 1) | (hits.all(-1).int() << 2))
        self.cur += 1
        return dict(hits=hits, cand=(tlp, tbi), old_pool=old_b_sc, cand_pool=cand_p)

    def state(self) -> dict:
        """The kernel's arrays: run_score, run_seq / pool_seq [B*nb, L], pool_score, pool_len, pool_fin, parent, tok, heur, flags."""
        R = self.B * self.nb
        return dict(run_score=self.r_sc.reshape(-1), run_seq=self.r_seq.reshape(R, self.L),
                    pool_seq=self.seqs.reshape(R, self.L), pool_score=self.b_sc.reshape(-1),
                    pool_len=(self.b_bi.reshape(R, -1) >= 0).sum(-1).int(), pool_fin=self.fin.reshape(-1).int(),
                    parent=self.parent, tok=self.tok, heur=self.heur.view(-1).int(), flags=self.flags)


# ------------------------------------------------------------------------------------------------------------------------
# self-tests

@pytest.mark.parametrize("V", [128256, 32000, 1024, 1000, 7, 1])
def test_log_softmax_bound_holds_on_fp32_emulation(V):
    g = torch.Generator().manual_seed(V)
    x = log_softmax_rows(V, g)
    got = emulate_log_softmax(x)
    frac = check_log_softmax(got, x)
    y, _ = log_softmax_ref(x)
    assert torch.equal(got[3], torch.full((V,), -math.log(V)).float()) or (got[3].double() + math.log(V)).abs().max() < 1e-5
    assert float(got[4, (V * 2) // 3]) == 0.0 and bool(torch.isneginf(y[4]).sum() == V - 1)
    print(f"V={V}: emulation uses {frac:.3f} of the bound")


def test_topk_exact_is_torch_topk_without_ties():
    g = torch.Generator().manual_seed(1)
    for N, K in ((128256 * 2, 16), (32000, 64), (1000, 4), (64, 64)):
        a = torch.randn(3, N, generator=g)
        v, i = topk_exact(a, K)
        ref = torch.topk(a, K)
        assert torch.equal(v, ref.values) and torch.equal(i, ref.indices)
    # ties: the lowest index first; -0.0 and +0.0 are one key
    a = torch.tensor([[1.0, 2.0, 1.0, -0.0, 2.0, 0.0, 1.0]])
    v, i = topk_exact(a, 5)
    assert i.tolist() == [[1, 4, 0, 2, 6]] and v.tolist() == [[2.0, 2.0, 1.0, 1.0, 1.0]]
    v, i = topk_exact(torch.tensor([[0.0, -1.0, -0.0]]), 2)
    assert i.tolist() == [[0, 2]] and torch.signbit(v[0, 1])


def test_hf_driver_reproduces_beam_search():
    """HFBeams fed the log-probs HF's own _beam_search used returns its sequences and scores."""
    from transformers import LlamaConfig, LlamaForCausalLM
    from transformers.generation.logits_process import LogitsProcessor, LogitsProcessorList
    V, nb, B, S, max_new = 96, 3, 2, 5, 6
    eos = [3, 11, 40]
    K = max(2, 1 + len(eos)) * nb
    for lpen, es in ((1.0, False), (0.0, True), (2.0, "never")):
        rec = []

        class Record(LogitsProcessor):
            def __call__(self, input_ids, scores):
                rec.append(scores.clone())
                return scores

        torch.manual_seed(0)
        hf = LlamaForCausalLM(LlamaConfig(vocab_size=V, hidden_size=16, intermediate_size=32, num_hidden_layers=1,
                                          num_attention_heads=2, num_key_value_heads=1, bos_token_id=None, eos_token_id=None,
                                          pad_token_id=None)).eval()
        with torch.no_grad():
            for p in hf.parameters():
                p.mul_(8.0)                          # peaked enough for the EOS ids to finish hypotheses
        ids = torch.randint(0, V, (B, S), generator=torch.Generator().manual_seed(2))
        with torch.no_grad():
            out = hf.generate(ids, num_beams=nb, length_penalty=lpen, early_stopping=es, num_return_sequences=nb,
                              eos_token_id=eos, pad_token_id=0, max_new_tokens=max_new, do_sample=False, output_scores=True,
                              return_dict_in_generate=True, logits_processor=LogitsProcessorList([Record()]))
        drv = HFBeams(ids, nb, V, K, max_new, eos, lpen, es)
        for lp in rec:
            assert drv.go
            drv.step(lp.float())
        assert not drv.go or len(rec) == max_new
        st = drv.state()
        width = out.sequences.shape[1]
        assert torch.equal(st["pool_seq"][:, :width], out.sequences), (lpen, es)
        assert torch.equal(st["pool_score"], out.sequences_scores.float()), (lpen, es)
