"""GPU: beam selection and the head's top-K / log-sum-exp epilogues on their own, against the fp64 beam rule.

- Epilogues (parseq_head_lse_bf16, parseq_head_topk_bf16): logits that fp32 holds exactly (small integers times 1/8, so
  every summation order gives the same bits) must give the numpy keys bit for bit, the tile maxima and target logits
  bit for bit, and tile sums within a stated fp32 bound of fp64; rows at or past M stay untouched.
- Searches driven from Python (parseq_beam_select): every step reads the state, evaluates beam_oracle's logits_fn on each
  active slot's prefix, uploads the rows (<= 128 classes) or runs the top-K epilogue (> 128), and selects.  On gapped
  rows (tests/selection_reference.py) the fp32 kernels must equal the fp64 rule bit for bit: each step against the rule
  applied to the kernel's own previous state, and the whole search against beam_oracle / lexicon_oracle.
- End to end with head.weight = 0: every logits row is the crafted head.bias, so beam_search, lexicon beam search,
  score and lexicon_decode must equal the fp64 oracles bit for bit through the engine's groups and super-chunks.
"""
import ctypes as ct

import numpy as np
import pytest
import torch

import beam_oracle as BO
import lexicon_oracle as LO
import selection_reference as SR

pytestmark = pytest.mark.gpu

ACTIVE, DONE, EMPTY = 0, 1, 2
SENT_F = 0x7fc0dead                 # a NaN payload no kernel produces
SENT_K = 0xdeadbeefdeadbeef


def _check(lib, rc):
    from parseq_b200.engine import check
    check(lib, rc)


def _p(t):
    return None if t is None else t.data_ptr()


def _bits(x: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def _same_f32(a, b) -> bool:
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


# ---------------------------------------------------------------- epilogues
def _head_topk(lib, A, W, bias, M, N, k, mask=None, mask_div=1, pad=64):
    T = (N + 127) // 128
    part = torch.full((M + pad, T, 2), 0.0, device="cuda")
    part.view(torch.int32).fill_(SENT_F)
    keys = torch.full((M + pad, T, 16), 0, dtype=torch.int64, device="cuda")
    keys.view(torch.int64).fill_(SENT_K - (1 << 64))
    _check(lib, lib.parseq_head_topk_bf16(A.data_ptr(), A.stride(0), W.data_ptr(), W.stride(0), _p(bias), M, N, A.shape[1],
                                          k, _p(mask), mask_div, part.data_ptr(), keys.data_ptr(), None))
    torch.cuda.synchronize()
    return part.cpu().numpy(), keys.cpu().numpy().view(np.uint64)


def _head_lse(lib, A, W, bias, M, N, tgt=None, pad=64):
    T = (N + 127) // 128
    part = torch.zeros((M + pad, T, 2), device="cuda")
    part.view(torch.int32).fill_(SENT_F)
    tl = torch.zeros(M + pad, device="cuda")
    tl.view(torch.int32).fill_(SENT_F)
    tg = None if tgt is None else torch.from_numpy(np.concatenate([tgt, np.zeros(pad, np.int32)])).cuda()
    _check(lib, lib.parseq_head_lse_bf16(A.data_ptr(), A.stride(0), W.data_ptr(), W.stride(0), _p(bias), M, N, A.shape[1],
                                         _p(tg), part.data_ptr(), _p(tl if tgt is not None else None), None))
    torch.cuda.synchronize()
    return part.cpu().numpy(), tl.cpu().numpy()


def _exact_problem(M, N, seed):
    """A [M, 64], W [N, 64] small integers (W / 8) and a bias of eighths: every logit and partial sum is exact in fp32.
    Ties: the values are coarse.  Non-finite columns: NaN at N - 2, +inf at N // 2 (when N > 200), a whole tile of -inf
    (the second, when there are three or more), -0 at column 3."""
    g = np.random.default_rng(seed)
    A = g.integers(-3, 4, (M, 64)).astype(np.float32)
    W = g.integers(-3, 4, (N, 64)).astype(np.float32) / 8
    bias = g.integers(-16, 17, N).astype(np.float32) / 8
    bias[g.random(N) < 0.05] = -np.inf
    bias[N - 2] = np.nan
    if N > 200:
        bias[N // 2] = np.inf
    if N > 256:
        bias[128:256] = -np.inf
    W[3] = 0
    bias[3] = -0.0
    with np.errstate(invalid="ignore"):
        v = A.astype(np.float64) @ W.astype(np.float64).T + bias.astype(np.float64)
    v = np.where(np.isnan(bias)[None, :], np.nan, v)
    tA = torch.from_numpy(A).to(torch.bfloat16).cuda()
    tW = torch.from_numpy(W).to(torch.bfloat16).cuda()
    return tA, tW, torch.from_numpy(bias).cuda(), v


def _masks(M, N, div, seed):
    """Allowlist rows for row r // div: random, plus rows that allow exactly the classes at the 31/32 and 127/128
    boundaries, allow nothing but EOS, and allow everything but the first tile's characters."""
    g = np.random.default_rng(seed)
    R = (M + div - 1) // div
    allowed = g.random((R, N)) < 0.5
    edge = np.zeros(N, dtype=bool)
    edge[[c for c in (31, 32, 127, 128, 159, 160, N - 1) if c < N]] = True
    allowed[0] = edge
    if R > 1:
        allowed[1] = False
    if R > 2:
        allowed[2] = True
        allowed[2, 1:128] = False
    allowed[:, 0] = True
    words = np.stack([SR.mask_words(a, N) for a in allowed])
    return allowed, words


# (N, M) pairs covering N in {95, 128, 129, 255, 256, 3001, 16384} and M in {1, 127, 129, 300, 4097}
EPI_SHAPES = [(95, 1), (95, 4097), (128, 127), (129, 129), (255, 300), (256, 1), (256, 4097), (3001, 300), (3001, 127),
              (16384, 129), (16384, 1)]
SUM_REL = 40 * 2.0 ** -23     # 2-ulp expf per term, <= 34 fp32 additions of terms <= 1, against a sum >= 1


def _check_partials(part, M, v, allowed, what):
    mx, s = SR.tile_partials(v, allowed)
    got_m, got_s = part[:M, :, 0], part[:M, :, 1]
    assert _same_f32(got_m, mx.astype(np.float32)), what
    nan = np.isnan(s)
    assert bool((np.isnan(got_s) == nan).all()), what
    ok = ~nan
    assert bool((np.abs(got_s[ok] - s[ok]) <= SUM_REL * np.maximum(s[ok], 1.0)).all()), what
    assert bool((got_s[ok][s[ok] == 0] == 0).all()), what         # an all-masked / all -inf tile is exactly (-inf, 0)
    assert bool((part[M:].view(np.uint32) == SENT_F).all()), what + ": rows past M written"


@pytest.mark.parametrize("shape", EPI_SHAPES, ids=lambda s: f"N{s[0]}-M{s[1]}")
def test_epilogues_on_exact_logits(lib, shape):
    N, M = shape
    A, W, bias, v = _exact_problem(M, N, N * 7 + M)
    T = (N + 127) // 128
    # log-sum-exp epilogue, with targets (some rows without one)
    g = np.random.default_rng(M + N)
    tgt = g.integers(0, N, M).astype(np.int32)
    tgt[g.random(M) < 0.2] = -1
    part, tl = _head_lse(lib, A, W, bias, M, N, tgt)
    _check_partials(part, M, v, None, "lse")
    rows = np.arange(M)
    want = np.where(tgt >= 0, v[rows, np.maximum(tgt, 0)], np.nan).astype(np.float32)
    has = tgt >= 0
    assert _same_f32(tl[:M][has], want[has])
    assert bool((_bits(tl[:M][~has]) == SENT_F).all()) and bool((_bits(tl[M:]) == SENT_F).all())
    part2, _ = _head_lse(lib, A, W, bias, M, N, None)
    assert np.array_equal(part2.view(np.uint32), part.view(np.uint32))
    # top-K epilogue: k beyond the allowed classes of a tile, every allowlist row layout
    for k in (1, 2, 5, 16):
        for div in (None, 1, 16, 26):
            if div is None:
                allowed, words = None, None
            else:
                am, w = _masks(M, N, div, k * 31 + div)
                allowed, words = am[np.arange(M) // div], torch.from_numpy(w.view(np.int32)).cuda()
            part, keys = _head_topk(lib, A, W, bias, M, N, k, words, div or 1)
            what = f"k={k} div={div}"
            _check_partials(part, M, v, allowed, what)
            ref = SR.topk_keys(v.astype(np.float32), allowed, k)
            assert np.array_equal(keys[:M, :, :k], ref[:, :, :k]), what
            assert bool((keys[M:] == SENT_K).all()), what + ": rows past M written"
    assert T >= 1


def test_epilogues_on_realistic_logits(lib):
    """bf16 A and W at K = 384 against fp64: each logit within the fp32 accumulation bound vb = 384 u sum |a w|
    (u = 2^-24), tile maxima within vb, tile log-sum-exp within 2 vb + the sum bound, and the keys: each listed value
    within vb of its class's fp64 logit, listed in fp64 order up to 2 vb, and no class left out that beats the last
    listed one by more than 2 vb."""
    M, N, K = 300, 3001, 384
    g = torch.Generator().manual_seed(5)
    A = torch.randn(M, K, generator=g).to(torch.bfloat16)
    W = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, generator=g)
    v = A.double() @ W.double().T + bias.double()
    vb = (384 * 2.0 ** -24 * (A.double().abs() @ W.double().abs().T) + 2.0 ** -24 * bias.double().abs()).numpy()
    v = v.numpy()
    part, keys = _head_topk(lib, A.cuda(), W.cuda(), bias.cuda(), M, N, 8)
    mx, s = SR.tile_partials(v)
    T = mx.shape[1]
    vbt = np.pad(vb, ((0, 0), (0, T * 128 - N))).reshape(M, T, 128).max(axis=2)
    assert bool((np.abs(part[:M, :, 0] - mx) <= vbt).all())
    lse32 = part[:M, :, 0].astype(np.float64) + np.log(part[:M, :, 1].astype(np.float64))
    assert bool((np.abs(lse32 - (mx + np.log(s))) <= 2 * vbt + SUM_REL).all())
    for r in range(0, M, 7):
        for t in range(T):
            ks = keys[r, t, :8]
            cls = SR.key_class(ks)
            val = SR.key_value(ks).astype(np.float64)
            assert bool((np.abs(val - v[r, cls]) <= vb[r, cls]).all())
            f = v[r, cls]
            assert bool((f[1:] <= f[:-1] + 2 * vbt[r, t]).all())
            lo, hi = t * 128, min(N, t * 128 + 128)
            out = np.setdiff1d(np.arange(lo, hi), cls)
            assert bool((v[r, out] <= f[-1] + 2 * vbt[r, t]).all())


def test_head_entry_points_reject_bad_arguments_on_the_host(lib):
    from parseq_b200.engine import BeamSelectArgsC
    buf = ct.c_float(0)
    for k in (0, 17):
        assert lib.parseq_head_topk_bf16(None, 64, None, 64, None, 1, 1, 64, k, None, 1, ct.addressof(buf),
                                         ct.addressof(buf), None) != 0
    assert lib.parseq_head_topk_bf16(None, 64, None, 64, None, 1, 1, 64, 1, ct.addressof(buf), 0, ct.addressof(buf),
                                     ct.addressof(buf), None) != 0
    assert lib.parseq_head_lse_bf16(None, 64, None, 64, None, 1, 1, 64, ct.addressof(buf), ct.addressof(buf), None,
                                    None) != 0
    ok = dict(logits=1, ntiles=1, batch=1, num_classes=95, beam_width=4, step=0, num_steps=26, ids_in=1, score_in=1,
              len_in=1, st_in=1, ids_out=1, score_out=1, len_out=1, st_out=1, parent=1, ids_ld=27, out_ids=1, out_len=1,
              out_score=1)
    bad = [dict(beam_width=0), dict(beam_width=17), dict(ntiles=2), dict(step=26), dict(step=-1), dict(ids_ld=26),
           dict(logits=None), dict(logits=None, keys=1, part=1, first_edge=1, edge_class=1, edge_child=1, terminal=1,
                                   node_out=1), dict(batch=0), dict(class_mask=1, mask_ld=2), dict(parent=None),
           dict(first_edge=1)]
    for b in bad:
        a = BeamSelectArgsC(**{**ok, **b})
        assert lib.parseq_beam_select(ct.byref(a), None) != 0, b
        assert lib.parseq_last_error()


# ---------------------------------------------------------------- searches driven from Python
class Lex:
    """A lexicon DAG on the device (parseq_lexicon_desc arrays) and its host copy for lexicon_oracle."""

    def __init__(self, first_edge, edge_class, edge_child, terminal):
        self.h = (np.asarray(first_edge, np.int32), np.asarray(edge_class, np.int32), np.asarray(edge_child, np.int32),
                  np.asarray(terminal, np.uint8))
        self.d = [torch.from_numpy(a).cuda() for a in self.h]
        self.children = {}
        for v in range(len(self.h[3])):
            self.children[v] = {int(self.h[1][j]): int(self.h[2][j]) for j in range(self.h[0][v], self.h[0][v + 1])}


def _selector_rows(lib, rows, C, mask_words, mask_div, K, part, keys, row_ids):
    """part / keys of logits rows through the top-K epilogue: one M = 1 GEMM per row with A = e_0 and W[:, 0] = the
    row, so that any value (NaN, +-inf) reaches the epilogue exactly."""
    A = torch.zeros((1, 64), dtype=torch.bfloat16, device="cuda")
    A[0, 0] = 1
    T = (C + 127) // 128
    for r, row in zip(row_ids, rows):
        W = torch.zeros((C, 64), dtype=torch.bfloat16)
        W[:, 0] = torch.from_numpy(np.asarray(row, np.float32)).to(torch.bfloat16)
        assert _same_f32(W[:, 0].float().numpy(), np.asarray(row, np.float32)), "rows must be bf16-exact"
        W = W.cuda()
        m = None if mask_words is None else mask_words[r // mask_div:]
        _check(lib, lib.parseq_head_topk_bf16(A.data_ptr(), 64, W.data_ptr(), 64, None, 1, C, 64, K, _p(m), 1,
                                              part[r].data_ptr(), keys[r].data_ptr(), None))
    assert part.shape[1] == T


def _step_reference(ids, score, length, st, node, rows_of, allowed, K, step, S, lex):
    """The rule applied to one image's state (fp64): the whole pool in slot order, stable-sorted (the first K are kept).
    Entries are (score, parent slot, class or -1, child node)."""
    pool = []
    for k in range(K):
        if st[k] == DONE:
            pool.append((float(score[k]), k, -1, -1))
        elif st[k] == ACTIVE:
            row = rows_of(k)
            a = SR.effective(allowed, len(row))
            lse = BO._lse([row[c] for c in range(len(row)) if a[c]])
            order = BO.row_order(list(row), a)
            if lex is not None:
                kids = lex.children[node[k]] if step + 1 < S else {}
                order = [c for c in order if (c == 0 and lex.h[3][node[k]]) or c in kids]
            for c in order[:K]:
                child = -1 if (lex is None or c == 0) else lex.children[node[k]][c]
                pool.append((float(score[k]) + (row[c] - lse), k, c, child))
    pool = [p for p in pool if p[0] != -np.inf]
    return sorted(pool, key=lambda p: BO.rank_key(p[0]))


def run_search(lib, fns, allows, C, K, S, layout, lex=None, roots=None, exact=True):
    """Beam search of len(fns) images through parseq_beam_select, checking every step; returns (ids [B, K, S],
    lengths [B, K], scores [B, K]) as numpy."""
    B = len(fns)
    R, ld, L = B * K, S + 2, S
    T = (C + 127) // 128
    wide = C > 128 and lex is None
    ids = [torch.zeros((R, ld), dtype=torch.int32, device="cuda") for _ in range(2)]
    ids[0][:, 0] = C
    ids[0][:, 1:] = C + 1
    score = [torch.full((R,), -np.inf, device="cuda") for _ in range(2)]
    length = [torch.full((R,), -1, dtype=torch.int32, device="cuda") for _ in range(2)]
    st = [torch.full((R,), EMPTY, dtype=torch.int32, device="cuda") for _ in range(2)]
    score[0][::K], length[0][::K], st[0][::K] = 0.0, 0, ACTIVE
    node = [torch.full((R,), -7, dtype=torch.int32, device="cuda") for _ in range(2)]
    parent = torch.full((R,), -7, dtype=torch.int32, device="cuda")
    out_ids = torch.full((R, S), -7, dtype=torch.int32, device="cuda")
    out_len = torch.full((R,), -7, dtype=torch.int32, device="cuda")
    out_score = torch.zeros(R, device="cuda")
    masked = any(a is not None for a in allows)
    mw = np.stack([SR.mask_words(a, C) for a in allows]) if masked else None
    mask = torch.from_numpy(mw.view(np.int32)).cuda() if masked else None
    nrows = B * L if layout == "vitstr" else R
    logits = torch.zeros((nrows, C), device="cuda")
    part = torch.zeros((nrows, T, 2), device="cuda")
    keys = torch.zeros((nrows, T, 16), dtype=torch.int64, device="cuda")
    if layout == "vitstr":                                   # the head once over every (image, position) row
        host = np.stack([fns[b].row([0] * t) for b in range(B) for t in range(L)])
        if wide:
            _selector_rows(lib, host, C, mask, L, K, part, keys, range(nrows))
        else:
            logits.copy_(torch.from_numpy(host.astype(np.float32)))
    lexd = lex.d if lex is not None else [None] * 4
    roots_d = None if roots is None else torch.tensor(roots, dtype=torch.int32, device="cuda")
    for step in range(S):
        cur, nxt = step & 1, (step & 1) ^ 1
        h_ids, h_sc, h_len, h_st = ids[cur].cpu().numpy(), score[cur].cpu().numpy(), length[cur].cpu().numpy(), st[cur].cpu().numpy()
        h_node = node[cur].cpu().numpy() if step > 0 else np.array([(roots[r // K] if roots else 0) for r in range(R)])
        prefix = {r: h_ids[r, 1:1 + h_len[r]].tolist() for r in range(R) if h_st[r] == ACTIVE}
        if layout == "parseq":
            act = sorted(prefix)
            host = [fns[r // K].row(prefix[r]) for r in act]
            if wide:
                _selector_rows(lib, host, C, mask, K, K, part, keys, act)
            elif act:
                hl = logits.cpu().numpy()
                hl[act] = np.stack(host).astype(np.float32)
                logits.copy_(torch.from_numpy(hl))
            row0, img_stride, slot_stride = 0, K, 1
        else:
            row0, img_stride, slot_stride = step, L, 0
        a = BeamSelectArgs(logits=None if wide else logits.data_ptr(), part=part.data_ptr(),
                           keys=keys.data_ptr() if wide else None, ntiles=T, row0=row0, img_stride=img_stride,
                           slot_stride=slot_stride, batch=B, num_classes=C, beam_width=K, step=step, num_steps=S,
                           class_mask=_p(mask), mask_ld=(C + 31) // 32, ids_in=ids[cur].data_ptr(),
                           score_in=score[cur].data_ptr(), len_in=length[cur].data_ptr(), st_in=st[cur].data_ptr(),
                           ids_out=ids[nxt].data_ptr(), score_out=score[nxt].data_ptr(), len_out=length[nxt].data_ptr(),
                           st_out=st[nxt].data_ptr(), parent=parent.data_ptr(), ids_ld=ld, out_ids=out_ids.data_ptr(),
                           out_len=out_len.data_ptr(), out_score=out_score.data_ptr(), first_edge=_p(lexd[0]),
                           edge_class=_p(lexd[1]), edge_child=_p(lexd[2]), terminal=_p(lexd[3]), roots=_p(roots_d),
                           node_in=node[cur].data_ptr(), node_out=node[nxt].data_ptr())
        _check(lib, lib.parseq_beam_select(ct.byref(a), None))
        torch.cuda.synchronize()
        n_ids, n_sc, n_len, n_st = ids[nxt].cpu().numpy(), score[nxt].cpu().numpy(), length[nxt].cpu().numpy(), st[nxt].cpu().numpy()
        n_par, n_node = parent.cpu().numpy(), node[nxt].cpu().numpy()
        for b in range(B):
            r0 = b * K

            def rows_of(k, b=b, r0=r0):
                return fns[b].row(h_ids[r0 + k, 1:1 + h_len[r0 + k]].tolist())
            ref = _step_reference(h_ids[r0:r0 + K], h_sc[r0:r0 + K], h_len[r0:r0 + K], h_st[r0:r0 + K],
                                  h_node[r0:r0 + K], rows_of, allows[b], K, step, S, lex)
            _check_step(b, step, S, K, r0, ref, h_ids, h_len, h_st, n_ids, n_sc, n_len, n_st, n_par, n_node, lex, exact)
    res = (out_ids.cpu().numpy().reshape(B, K, S), out_len.cpu().numpy().reshape(B, K), out_score.cpu().numpy().reshape(B, K))
    last = S & 1
    fl, fs = length[last].cpu().numpy().reshape(B, K), score[last].cpu().numpy().reshape(B, K)
    fi = ids[last].cpu().numpy().reshape(B, K, ld)
    assert np.array_equal(res[1], fl) and _same_f32(res[2], fs)
    for b in range(B):
        for k in range(K):
            n = fl[b, k]
            want = np.zeros(S, np.int32)
            if n > 0:
                want[:n] = fi[b, k, 1:1 + n]
            assert res[0][b, k].tolist() == want.tolist(), (b, k)
    return res


def BeamSelectArgs(**kw):
    from parseq_b200.engine import BeamSelectArgsC
    return BeamSelectArgsC(**kw)


def _check_step(b, step, S, K, r0, ref, h_ids, h_len, h_st, n_ids, n_sc, n_len, n_st, n_par, n_node, lex, exact):
    """The kernel's new state of image b against the rule applied to its old state.  Exact (gapped or non-finite rows):
    every slot bit for bit.  Otherwise (bf16 rows): each kept entry is in the fp64 pool with a score within TOL of it, in
    fp64 order up to 2 TOL, and nothing left out beats the last kept entry by more than 2 TOL.  Always: a kept slot's ids
    are its parent's ids plus its class at position step + 1."""
    what = (b, step)
    got = []
    for k in range(K):
        r = r0 + k
        p = n_par[r] - r0
        assert 0 <= p < K, what
        if n_st[r] == EMPTY:
            assert n_len[r] == -1 and n_sc[r] == -np.inf and p == k, what
            assert n_ids[r].tolist() == h_ids[r].tolist(), what
            continue
        c = -1 if h_st[r0 + p] == DONE else int(n_ids[r, step + 1])
        want = h_ids[r0 + p].copy()
        if c >= 0:
            want[step + 1] = c
        assert n_ids[r].tolist() == want.tolist(), what           # the depth >= 2 K/V gather relies on this
        ln = h_len[r0 + p] if c < 0 else (step if c == 0 else step + 1)
        assert n_len[r] == ln, what
        assert n_st[r] == (DONE if c <= 0 or step + 1 == S else ACTIVE), what
        got.append((float(n_sc[r]), p, c, int(n_node[r]) if lex is not None else -1))
    assert len(got) == min(K, len(ref)), (what, got, ref[:K])
    if exact:
        for g, e in zip(got, ref[:K]):
            assert g[1:3] == e[1:3], (what, got, ref[:K])
            assert _same_f32(g[0], e[0]), (what, got, ref[:K])
            if lex is not None:
                assert g[3] == e[3], (what, got, ref[:K])
        return
    # bf16 rows: TOL covers the fp32 rounding of the log-sum-exp (<= C / 32 + 7 additions) and of the two additions
    full = {(e[1], e[2]): e[0] for e in ref}
    f64 = []
    for g in got:
        assert (g[1], g[2]) in full, (what, g)
        f64.append(full[(g[1], g[2])])
        assert abs(g[0] - f64[-1]) <= TOL * (1 + abs(f64[-1])), (what, g, f64[-1])
    kept = {(g[1], g[2]) for g in got}
    last = min(f64)
    for e in ref:
        if e[0] > last + 2 * TOL * (1 + abs(last)):
            assert (e[1], e[2]) in kept, (what, e)
    for i in range(1, len(f64)):
        assert f64[i] <= f64[i - 1] + 2 * TOL * (1 + abs(f64[i])), what


TOL = 2e-5


def _oracle_equal(res, fns, allows, K, S, lex=None, roots=None):
    ids, lens, scores = res
    for b in range(len(fns)):
        if lex is None:
            want = BO.beam_search(fns[b], K, S, allows[b])
        else:
            want = LO.lexicon_beam_search(fns[b], K, S, *lex.h, root=roots[b] if roots else 0, allowed=allows[b])
        for k in range(K):
            if k < len(want):
                assert lens[b, k] == len(want[k][0]) and ids[b, k, :lens[b, k]].tolist() == want[k][0], (b, k)
                assert _same_f32(scores[b, k], np.float32(want[k][1])), (b, k, scores[b, k], want[k][1])
            else:
                assert lens[b, k] == -1 and scores[b, k] == -np.inf, (b, k)


@pytest.mark.parametrize("case", SR.SEARCH_CASES, ids=lambda c: f"C{c[0]}-K{c[1]}-S{c[2]}-{c[3]}")
def test_gapped_search_equals_the_fp64_rule_bit_for_bit(lib, case):
    C, K, S, layout, seed = case
    allows = SR.case_allowlists(C, seed)
    fns = SR.case_logits_fns(C, seed, layout)
    res = run_search(lib, fns, allows, C, K, S, layout)
    _oracle_equal(res, fns, allows, K, S)


@pytest.mark.parametrize("case", [(95, 8, 26, "parseq", 21), (129, 4, 12, "parseq", 22), (3001, 6, 8, "vitstr", 23),
                                  (128, 16, 10, "vitstr", 24)], ids=lambda c: f"C{c[0]}-K{c[1]}-{c[3]}")
def test_nonfinite_rows_follow_the_discrete_rules(lib, case):
    """A third of the rows carry a NaN or +inf at an allowed class: their children score NaN, NaN logits expand first,
    NaN ranks after every number."""
    C, K, S, layout, seed = case
    allows = SR.case_allowlists(C, seed)
    fns = SR.case_logits_fns(C, seed, layout, nonfinite=0.35)
    res = run_search(lib, fns, allows, C, K, S, layout)
    assert np.isnan(res[2]).any()
    _oracle_equal(res, fns, allows, K, S)


@pytest.mark.parametrize("case", [(3, 3, 26, "parseq"), (95, 16, 26, "parseq"), (129, 8, 26, "parseq"),
                                  (3001, 5, 12, "parseq"), (128, 4, 26, "vitstr"), (3001, 16, 8, "vitstr")],
                         ids=lambda c: f"C{c[0]}-K{c[1]}-{c[3]}")
def test_bf16_random_rows_within_the_fp32_bound(lib, case):
    C, K, S, layout = case
    fns = [SR.bf16_logits_fn(C, 40 + b, layout == "vitstr") for b in range(3)]
    allows = SR.case_allowlists(C, 40)[:3]
    run_search(lib, fns, allows, C, K, S, layout, exact=False)


def _trie_words(g, C, n, maxlen, alphabet=None):
    cls = np.arange(1, C) if alphabet is None else np.asarray(alphabet)
    return [g.choice(cls, size=int(g.integers(1, maxlen + 1))).tolist() for _ in range(n)]


def _lex_cases():
    from parseq_b200.lexicon import build_trie
    g = np.random.default_rng(7)
    out = []
    # per-image roots of a trie forest; image 1's list holds "" (a terminal root); words longer than num_steps - 1
    rows = [_trie_words(g, 95, 30, 9, range(1, 6)), _trie_words(g, 95, 20, 4) + [[]], _trie_words(g, 95, 60, 12, range(1, 4)),
            [[1, 2], [1, 2, 3, 4, 5, 6, 7, 8, 9, 10]]]
    out.append(("forest-C95", 95, 8, 7, Lex(*build_trie(rows)), [0, 1, 2, 3]))
    # a node with more than 32 edges (40 classes spread over the 3001 classes, across word and tile boundaries)
    wide = sorted(set(g.choice(np.arange(1, 3001), 38, replace=False).tolist()) | {31, 32, 127, 128})
    rows = [[[c] for c in wide] + [[c, 5] for c in wide[:10]] + [[wide[3], 7, 9]]]
    out.append(("wide-node-C3001", 3001, 16, 4, Lex(*build_trie(rows)), [0, 0, 0, 0]))
    # a DAG with shared suffix nodes: 0 -1-> 1, 0 -2-> 2, 0 -3-> 3; 1 -4-> 4, 2 -4-> 4, 2 -5-> 5, 3 -5-> 5;
    # 4 (terminal) -6-> 6; 5 terminal; 6 terminal -7-> 7 (terminal)
    fe = [0, 3, 4, 6, 7, 8, 8, 9, 9]
    ec = [1, 2, 3, 4, 4, 5, 5, 6, 7]
    ch = [1, 2, 3, 4, 4, 5, 5, 6, 7]
    term = [0, 0, 0, 0, 1, 1, 1, 1]
    out.append(("dag-C95", 95, 4, 5, Lex(fe, ec, ch, term), [0, 2, 0, 3]))
    out.append(("dag-C3001-K16", 3001, 16, 26, Lex(fe, ec, ch, term), None))
    return out


@pytest.mark.parametrize("idx", range(4), ids=["forest-C95", "wide-node-C3001", "dag-C95", "dag-C3001-K16"])
def test_lexicon_search_equals_the_fp64_rule_bit_for_bit(lib, idx):
    name, C, K, S, lex, roots = _lex_cases()[idx]
    allows = SR.case_allowlists(C, 50 + idx)
    if C > 128:
        allows[1] = None                   # the random half leaves too few of the wide node's classes
    fns = [SR.gapped_logits_fn(C, 500 + 10 * idx + b, a, levels=2) for b, a in enumerate(allows)]
    res = run_search(lib, fns, allows, C, K, S, "parseq", lex=lex, roots=roots)
    _oracle_equal(res, fns, allows, K, S, lex=lex, roots=roots)
    assert (res[1] >= 0).any()


# ---------------------------------------------------------------- end to end with head.weight = 0
def _e2e_model(experiment, C, bias, dec_depth=1, mll=25):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    n_extra = C - 95
    extra = {} if experiment == "vitstr" else {"dec_depth": dec_depth}
    cfg = make_config_long(experiment, mll, n_extra, **extra)
    sd = init_state_dict(cfg, 3, sharp=2.0)
    sd["head.weight"] = torch.zeros_like(sd["head.weight"])
    sd["head.bias"] = torch.from_numpy(np.asarray(bias, np.float32))
    cs = charset(n_extra)
    m = create_model(experiment, charset_train=cs, charset_test=cs, max_label_length=mll, **extra)
    (m if experiment == "vitstr" else m.model).load_state_dict(sd)
    m = m.eval().to("cuda")
    m.model.set_engine_option("max_batch", 16)      # 20 images: two super-chunks
    if experiment != "vitstr":
        m.model.set_engine_option("dec_chunk", 16)  # 16 // K images per decoder group
    return cfg, cs, m


E2E_CASES = [("parseq", 95, 1, None, 5), ("parseq", 95, 2, None, 3), ("parseq", 128, 1, None, 8),
             ("parseq", 129, 2, 12, 4), ("parseq", 3001, 1, 8, 16), ("parseq", 16384, 1, 3, 6), ("vitstr", 95, 1, None, 5),
             ("vitstr", 129, 1, 10, 16), ("vitstr", 3001, 1, 6, 3), ("vitstr", 16384, 1, 3, 4)]


def _allow_mask(allows, C, N):
    rows = [allows[b % len(allows)] for b in range(N)]
    words = np.stack([SR.mask_words(a, C) for a in rows])
    return rows, torch.from_numpy(words.view(np.int32)).cuda()


@pytest.mark.parametrize("case", E2E_CASES, ids=lambda c: f"{c[0]}-C{c[1]}-depth{c[2]}-K{c[4]}")
def test_end_to_end_beam_and_lexicon_search_and_scores_with_a_constant_head(lib, case):
    from parseq_b200.lexicon import build_trie
    from parseq_b200.weights import synth_images
    experiment, C, depth, max_length, K = case
    bias, allows = SR.e2e_bias(C)
    cfg, cs, m = _e2e_model(experiment, C, bias, depth)
    N = 20
    x = synth_images(cfg, N, 9).cuda()
    S = (cfg.max_label_length if max_length is None else min(max_length, cfg.max_label_length)) + 1
    rows, mask = _allow_mask(allows, C, N)
    fn = lambda ps: [bias] * len(ps)
    with torch.inference_mode():
        ids, lens, scores = m.model.beam_search(x, K, max_length, class_mask=mask)
    res = (ids.cpu().numpy(), lens.cpu().numpy(), scores.cpu().numpy())
    _oracle_equal(res, [fn] * N, rows, K, S)
    # lexicon beam search: per-image word lists (one holds ""), words too long for max_length included
    g = np.random.default_rng(C + depth)
    top = [5, 9, 1, 2, 3] + g.integers(1, C, 4).tolist()
    word_rows = [[g.choice(top, size=int(g.integers(0, 6))).tolist() for _ in range(12)] for _ in range(N)]
    lex_strings = [["".join(cs[c - 1] for c in w) for w in r] for r in word_rows]
    trie = Lex(*build_trie(word_rows))
    with torch.inference_mode():
        lx = m.compile_lexicon(lex_strings)
        ids, lens, scores = m.model.beam_search(x, K, max_length, class_mask=mask, lexicon=lx, roots=lx.roots_for(N))
    res = (ids.cpu().numpy(), lens.cpu().numpy(), scores.cpu().numpy())
    _oracle_equal(res, [fn] * N, rows, K, S, lex=trie, roots=list(range(N)))
    # score / lexicon_decode: sum of bias[t_i] - max(bias) over the label's characters and its EOS (no allowlist)
    mll = cfg.max_label_length
    words = [w for w in word_rows[0] if len(w) <= mll][:6] + [[5] * min(mll, 30)]
    strings = ["".join(cs[c - 1] for c in w) for w in words]
    with torch.inference_mode():
        sc = m.score(x, strings).cpu().numpy()
        labels, lp = m.lexicon_decode(x, strings)
    want = np.array([BO.sequence_logprob(fn, w, mll + 1) for w in words], dtype=np.float32)
    assert _same_f32(want, [sum(bias[t] - np.max(bias) for t in w + [0]) for w in words])
    for b in range(N):
        assert _same_f32(sc[b], want), b
        assert labels[b] == strings[int(np.argmax(want))] and _same_f32(lp[b].item(), want.max()), b


@pytest.mark.parametrize("case", [("parseq", 95), ("parseq", 3001), ("vitstr", 129)], ids=lambda c: f"{c[0]}-C{c[1]}")
def test_end_to_end_nonfinite_head_follows_the_discrete_rules(lib, case):
    """NaN and +inf bias classes: every log-sum-exp is NaN, so every score is NaN; NaN classes expand first (lower
    class first), then the logits in order; the pool keeps its slot order among NaN scores.  An allowlist that masks the
    NaN and +inf classes gives finite scores again."""
    from parseq_b200.weights import synth_images
    experiment, C = case
    bias, _ = SR.e2e_bias(C)
    bias = bias.copy()
    bias[[7, 40]] = np.nan
    bias[60] = np.inf
    cfg, cs, m = _e2e_model(experiment, C, bias)
    allow = np.ones(C, dtype=bool)
    allow[[7, 40, 60]] = False
    allows = [None, allow]
    N, K, max_length = 4, 5, 6
    rows, mask = _allow_mask(allows, C, N)
    x = synth_images(cfg, N, 9).cuda()
    with torch.inference_mode():
        ids, lens, scores = m.model.beam_search(x, K, max_length, class_mask=mask)
    res = (ids.cpu().numpy(), lens.cpu().numpy(), scores.cpu().numpy())
    assert np.isnan(res[2][0]).all() and np.isfinite(res[2][1]).all()
    _oracle_equal(res, [lambda ps: [bias] * len(ps)] * N, rows, K, max_length + 1)
