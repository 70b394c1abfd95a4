"""GPU: non-finite values.  Every greedy argmax of the engine follows torch.argmax (the first NaN, else the first maximum,
+inf counting as a maximum, -0.0 == +0.0, a row of -inf gives 0), so an id fed back into the AR loop is always a class of
the head.  The fused postprocess follows `logits.softmax(-1)` -> `Tokenizer.decode` -> `prob.prod()`: a row whose softmax
is all NaN gives id 0 (EOS) with probability NaN.  A crop of NaN or +inf pixels must not change any other image of its
batch, nor an image of a later call on the same handle, at any image-token count T.

Expected values always come from torch on the CPU (the reference pipeline or the fp32 ParseqOracle), never from a table
written by hand."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")


def _charset(C):
    from parseq_b200.config import CHARSET_94
    return CHARSET_94 + "".join(chr(0x4E00 + i) for i in range(C - 95))          # C head classes = charset + EOS


def _bits(t):
    """Bitwise view for comparisons that must treat NaN as equal to the same NaN."""
    return t.contiguous().view(torch.int32)


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _nan_equal_close(a, b, rtol=1e-5, atol=0.0):
    if a.shape != b.shape or not torch.equal(torch.isnan(a), torch.isnan(b)):
        return False
    f = ~torch.isnan(a)
    return torch.allclose(a[f], b[f], rtol=rtol, atol=atol, equal_nan=False)


# ---------------------------------------------------------------------------------------------------------------------
# stand-alone postprocess on crafted logits

def _places(C):
    return [0, 31, 32, 33, C - 1]        # different lanes, the same lane (0 / 32), neighbours, the last column


def _crafted_rows(C, g):
    """(name, row) pairs: every special pattern at every placement (pairs in both index orders where it matters)."""
    P = _places(C)
    pairs = [(a, b) for a in P for b in P if a < b]
    base = lambda: torch.randn(C, generator=g)                                    # noqa: E731
    rows = []
    for a in P:
        r = base(); r[a] = NAN; rows.append((f"nan@{a}", r))
        r = torch.full((C,), -INF); r[a] = 1.5; rows.append((f"only_finite@{a}", r))
        r = base(); r[a] = INF; rows.append((f"inf@{a}", r))
    for a, b in pairs:
        r = base(); r[a] = NAN; r[b] = NAN; rows.append((f"nan@{a},{b}", r))
        r = base(); r[a] = INF; r[b] = INF; rows.append((f"inf@{a},{b}", r))
        r = base(); r[a] = INF; r[b] = NAN; rows.append((f"inf@{a},nan@{b}", r))
        r = base(); r[a] = NAN; r[b] = INF; rows.append((f"nan@{a},inf@{b}", r))
        r = -1.0 - base().abs(); r[a] = -0.0; r[b] = 0.0; rows.append((f"-0@{a},+0@{b}", r))
        r = -1.0 - base().abs(); r[a] = 0.0; r[b] = -0.0; rows.append((f"+0@{a},-0@{b}", r))
    for j in (0, 31, 33, C - 34):
        for k in (j + 1, j + 32):
            r = base(); r[j] = r[k] = 9.0; rows.append((f"tie@{j},{k}", r))
    rows.append(("all_-inf", torch.full((C,), -INF)))
    rows.append(("all_nan", torch.full((C,), NAN)))
    rows.append(("all_+inf", torch.full((C,), INF)))
    return rows


def _postprocess(logits):
    from parseq_b200.engine import check, load_library
    lib = load_library()
    B, L, C = logits.shape
    x = logits.cuda().contiguous()
    ids = torch.empty((B, L), dtype=torch.int32, device="cuda")
    lengths = torch.empty((B,), dtype=torch.int32, device="cuda")
    conf = torch.empty((B,), dtype=torch.float32, device="cuda")
    check(lib, lib.parseq_postprocess(x.data_ptr(), B, L, C, 0, ids.data_ptr(), lengths.data_ptr(), conf.data_ptr(),
                                      ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return ids.cpu(), lengths.cpu(), conf.cpu()


def _reference_postprocess(logits, tok):
    """base.py:132-142 on the CPU: softmax -> Tokenizer.decode (greedy max, cut at the first EOS) -> prod."""
    probs = logits.softmax(-1)
    ids = probs.max(-1).indices
    labels, p = tok.decode(probs)
    L = logits.shape[1]
    lengths = torch.tensor([(r == 0).nonzero()[0].item() if bool((r == 0).any()) else L for r in ids])
    conf = torch.stack([q.prod() for q in p])
    return ids, lengths, labels, conf


@pytest.mark.parametrize("C", [95, 3001, 16384])
def test_postprocess_nonfinite_rows_match_softmax_decode(C):
    from parseq_b200.tokenizer import Tokenizer
    g = torch.Generator().manual_seed(C)
    rows = _crafted_rows(C, g)
    L = 4
    # each crafted row sits at one position of its own image, the other positions are finite rows whose EOS logit is low
    # (so that an image's length is set by the crafted row or runs to L); the position cycles through 0..L-1
    B = len(rows)
    logits = torch.randn((B, L, C), generator=g)
    logits[..., 0] -= 20.0
    for b, (_, r) in enumerate(rows):
        logits[b, b % L] = r
    ids, lengths, conf = _postprocess(logits)
    tok = Tokenizer(_charset(C))
    r_ids, r_len, r_labels, r_conf = _reference_postprocess(logits, tok)
    for b, (name, _) in enumerate(rows):
        s = b % L
        assert ids[b, s].item() == r_ids[b, s].item(), (name, ids[b, s].item(), r_ids[b, s].item())
    assert torch.equal(ids.long(), r_ids)
    assert torch.equal(lengths.long(), r_len)
    labels = [tok._ids2tok(row[:n], True) for row, n in zip(ids.tolist(), lengths.tolist())]
    assert labels == r_labels
    bad = [(rows[b][0], conf[b].item(), r_conf[b].item()) for b in range(B)
           if not _nan_equal_close(conf[b:b + 1], r_conf[b:b + 1].float(), rtol=1e-4)]
    assert not bad, bad
    assert bool(torch.isnan(conf).any()) and bool(torch.isfinite(conf).any())


def test_argmax_order_expectations_are_torchs():
    """The semantics the kernels implement, stated on torch itself (CPU), so a change of torch shows up here."""
    t = torch.tensor
    assert t([1.0, NAN, 3.0, NAN]).argmax().item() == 1
    assert t([1.0, NAN, 3.0, NAN]).softmax(-1).max(-1).indices.item() == 0
    assert t([1.0, 5.0, INF, INF]).argmax().item() == 2
    assert t([1.0, 5.0, INF, INF]).softmax(-1).max(-1).indices.item() == 0
    assert t([-INF] * 3).argmax().item() == 0
    assert t([-1.0, -0.0, 0.0]).argmax().item() == 1 and t([-1.0, 0.0, -0.0]).argmax().item() == 1


# ---------------------------------------------------------------------------------------------------------------------
# in-model argmax sites: non-finite head biases keep every id inside the head

def _model(experiment, C, seed, sd_edit, **kw):
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    over = {} if C == 95 else {"charset_train": _charset(C)}
    cfg = make_config(experiment, **over, **{k: v for k, v in kw.items() if k in ("enc_depth", "img_size", "patch_size")})
    sd = init_state_dict(cfg, seed)
    sd_edit(sd)
    m = create_model(experiment, **over, **kw)
    (m if experiment == "vitstr" else m.model).load_state_dict(sd)
    return cfg, sd, m.eval().to("cuda")


def _bias(values):
    def edit(sd):
        b = sd["head.bias"].clone()
        for k, v in values.items():
            b[k] = v
        sd["head.bias"] = b
    return edit


def _replay_forcing(m, ids, decode_ar, refine_iters, k):
    """Teacher forcing that replays `k` as every decision: AR context [BOS, k, k, ...], refine contexts likewise."""
    B, L = ids.shape
    forced = forced_refine = None
    if decode_ar:
        forced = torch.full((B, L), k, dtype=torch.int32)
        forced[:, 0] = m.bos_id
    if refine_iters:
        forced_refine = torch.full((refine_iters, B, L), k, dtype=torch.int32)
        forced_refine[:, :, 0] = m.bos_id
    return forced, forced_refine


# (ar_kernel, ar_cluster_size, batch): the cluster kernel with clusters of 8 and 6, its head-split regime (one image),
# the grid-barrier kernel (<= 128 classes only) and the chain of separate kernels
AR_REGIMES = [(2, 8, 5), (2, 6, 5), (2, 8, 1), (1, 0, 5), (0, 0, 5)]
# C = 3001: clusters of 8 own 376 classes each, clusters of 6 own 504 (the comment before TIES in
# test_gpu_large_charset.py): k in a non-zero slice, at the first class of slice 1 (8) / slice 1 (6), in the last slice
NAN_COLUMNS = {95: [0, 31, 94], 3001: [400, 376, 504, 3000]}


def _check_all_ids(m, x, decode_ar, refine_iters, want, replay_k=None):
    m.model.decode_ar, m.model.refine_iters = decode_ar, refine_iters
    with torch.inference_mode():
        logits, ids = m.model.forward(m.tokenizer, x, 25, return_ids=True)
        assert bool((ids == want).all()), (decode_ar, refine_iters, ids.unique().tolist())
        forced, forced_refine = _replay_forcing(m, ids, decode_ar, refine_iters, want if replay_k is None else replay_k)
        again = m.model.forward(m.tokenizer, x, 25, forced_ids=forced, forced_refine=forced_refine)
    assert _same_bits(again, logits)
    return logits


@pytest.mark.parametrize("C,k", [(C, k) for C, ks in NAN_COLUMNS.items() for k in ks])
def test_nan_head_column_is_every_id_and_replays_bit_identically(C, k):
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", C, 21, _bias({k: NAN}))
    for impl, cs, B in AR_REGIMES:
        if impl == 1 and C > 128:
            continue
        m.model.set_engine_option("ar_kernel", impl)
        if cs:
            m.model.set_engine_option("ar_cluster_size", cs)
        x = synth_images(cfg, B, 70 + B).cuda()
        logits = _check_all_ids(m, x, True, 1, k)
        assert bool(torch.isnan(logits[..., k]).all()) and bool(torch.isfinite(logits[..., :k]).all())
        if impl == 2 and cs == 8 and B == 1:
            assert m.model.engine().debug_int("ar_last_per") == 1
        if impl == 2:
            assert m.model.engine().debug_int("ar_last_cluster_size") == cs
    x = synth_images(cfg, 5, 75).cuda()
    _check_all_ids(m, x, False, 2, k)                       # NAR + 2 refine


@pytest.mark.parametrize("C,k", [(95, 0), (95, 94), (3001, 400), (3001, 3000)])
def test_nan_head_column_vitstr(C, k):
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("vitstr", C, 22, _bias({k: NAN}))
    x = synth_images(cfg, 3, 76).cuda()
    with torch.inference_mode():
        logits, ids = m.model.forward_tokens(x, 25, return_ids=True)
    assert bool((ids == k).all()) and bool(torch.isnan(logits[..., k]).all())


@pytest.mark.parametrize("C,a,b", [(95, 31, 32), (95, 3, 94), (3001, 100, 2500), (3001, 376, 377)])
def test_inf_biases_first_wins_and_nan_after_inf_wins(C, a, b):
    from parseq_b200.weights import synth_images
    for bias, want in (({a: INF, b: INF}, a), ({a: INF, b: NAN}, b)):
        cfg, sd, m = _model("parseq", C, 23, _bias(bias))
        for impl, cs, B in AR_REGIMES:
            if impl == 1 and C > 128:
                continue
            m.model.set_engine_option("ar_kernel", impl)
            if cs:
                m.model.set_engine_option("ar_cluster_size", cs)
            _check_all_ids(m, synth_images(cfg, B, 80 + B).cuda(), True, 1, want)
        _check_all_ids(m, synth_images(cfg, 4, 85).cuda(), False, 2, want)


# ---------------------------------------------------------------------------------------------------------------------
# per-image isolation of non-finite crops

# T -> (experiment, img_size, patch_size)
GEOMETRIES = {
    32: ("parseq", (16, 64), (4, 8)),
    49: ("parseq", (28, 28), (4, 4)),
    100: ("parseq", (40, 80), (4, 8)),
    128: ("parseq", (32, 128), (4, 8)),
    130: ("parseq", (40, 104), (4, 8)),
    196: ("parseq", (224, 224), (16, 16)),
    240: ("parseq", (48, 160), (4, 8)),
}
# (ar_kernel, ar_cluster_size) of the AR loop; NAR runs no AR loop
AR_IMPLS = [(2, 8), (2, 6), (1, 0), (0, 0)]


def _isolation_model(T, C=95, seed=30):
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    exp, img, patch = GEOMETRIES[T]
    over = dict(img_size=img, patch_size=patch, enc_depth=2)
    if C != 95:
        over["charset_train"] = _charset(C)
    cfg = make_config(exp, **over)
    assert cfg.num_patches == T
    sd = init_state_dict(cfg, seed, sharp=4.0)

    def make():
        m = create_model(exp, **over)
        m.model.load_state_dict(sd)
        return m.eval().to("cuda")
    return cfg, sd, make


def _dirty(x, bad):
    y = x.clone()
    for i, v in bad.items():
        y[i] = v
    return y


def _run(m, x, ar, ri):
    m.model.decode_ar, m.model.refine_iters = ar, ri
    with torch.inference_mode():
        lg, ids = m.model.forward(m.tokenizer, x.cuda(), 25, return_ids=True)
    return lg.cpu(), ids.cpu()


def _check_isolation(cfg, sd, make, ar, ri, impls, B=12, max_batch=None):
    from oracle.parseq_oracle import ParseqOracle
    from parseq_b200.weights import synth_images
    m = make()
    if max_batch is not None:
        m.model.set_engine_option("max_batch", max_batch)
    x = synth_images(cfg, B, 90 + B)
    mid = B // 2
    oracle = ParseqOracle(cfg, sd, "fp32")
    failures = []
    for fills in ((NAN, INF, NAN), (INF, NAN, INF)):
        bad = {0: fills[0], mid: fills[1], B - 1: fills[2]}
        xd = _dirty(x, bad)
        o = oracle.forward(xd[list(bad)], 25, ar, ri)
        for impl, cs in impls:
            tag = (impl, cs, fills[0])
            m.model.set_engine_option("ar_kernel", impl)
            if cs:
                m.model.set_engine_option("ar_cluster_size", cs)
            lc, ic = _run(m, x, ar, ri)
            ld, idd = _run(m, xd, ar, ri)
            good = [i for i in range(B) if i not in bad]
            if not (_same_bits(ld[good], lc[good]) and torch.equal(idd[good], ic[good])):
                rows = [i for i in good if not _same_bits(ld[i], lc[i])]
                failures.append(("clean rows moved", tag, rows))
            for j, i in enumerate(bad):
                if not (_nan_equal_close(ld[i], o.logits[j].float(), rtol=0, atol=2e-2)
                        and torch.equal(idd[i].long(), o.ids[j])):
                    failures.append(("bad row differs from the oracle", tag, i))
            labels, confs = m.postprocess(ld[list(bad)].cuda())
            r_labels, r_probs = m.tokenizer.decode(o.logits.float().softmax(-1))
            r_conf = torch.stack([p.prod() for p in r_probs])
            if labels != r_labels or not _nan_equal_close(torch.tensor(confs), r_conf.float()):
                failures.append(("bad row label / confidence", tag, labels, confs))
    return m, failures


@pytest.mark.parametrize("mode", ["ar1", "nar2"])
@pytest.mark.parametrize("T", sorted(GEOMETRIES))
def test_nonfinite_crops_do_not_leak_into_other_images(T, mode):
    cfg, sd, make = _isolation_model(T)
    ar, ri = (True, 1) if mode == "ar1" else (False, 2)
    _, failures = _check_isolation(cfg, sd, make, ar, ri, AR_IMPLS if ar else AR_IMPLS[:1])
    assert not failures, failures


@pytest.mark.parametrize("T", sorted(GEOMETRIES))
def test_nonfinite_crop_does_not_leak_into_a_later_call(T):
    """The cross K/V cache keeps a previous call's rows: a NaN crop at index 5 of an 8-image call must not reach image 4
    of a following 5-image call on the same handle."""
    from parseq_b200.weights import synth_images
    cfg, sd, make = _isolation_model(T)
    x8 = _dirty(synth_images(cfg, 8, 95), {5: NAN})
    x5 = synth_images(cfg, 5, 96)
    failures = []
    for mode in ((True, 1), (False, 2)):
        for impl, cs in (AR_IMPLS if mode[0] else AR_IMPLS[:1]):
            ms = []
            for _ in range(2):
                m = make()
                m.model.set_engine_option("ar_kernel", impl)
                if cs:
                    m.model.set_engine_option("ar_cluster_size", cs)
                ms.append(m)
            _run(ms[0], x8, *mode)
            after = _run(ms[0], x5, *mode)
            fresh = _run(ms[1], x5, *mode)
            if not (_same_bits(after[0], fresh[0]) and torch.equal(after[1], fresh[1])):
                failures.append((mode, impl, cs))
    assert not failures, failures


def test_nonfinite_crops_wide_head_t196():
    cfg, sd, make = _isolation_model(196, C=3001)
    _, failures = _check_isolation(cfg, sd, make, True, 1, [(2, 8), (2, 6), (0, 0)], B=10)
    assert not failures, failures


@pytest.mark.parametrize("T", [32, 49, 130])
def test_nonfinite_crops_full_workspace(T):
    """B = max_batch: the last image's K/V box runs past the end of the cache."""
    cfg, sd, make = _isolation_model(T)
    _, failures = _check_isolation(cfg, sd, make, True, 1, AR_IMPLS, B=12, max_batch=12)
    assert not failures, failures
