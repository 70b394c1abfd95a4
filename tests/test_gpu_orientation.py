"""GPU: per-crop rotations and the orientation search (parseq_forward_crops_oriented).

  * a `rotation` list reads every crop exactly as a call at that crop's rotation (logits, ids, maps, and the step
    count of the per-crop calls' maximum), for CUDA and host crops and across super-chunks, with the launches of a
    uniform call;
  * the search returns, crop by crop, the engine's own forward at the orientation tests/orientation_oracle.py picks
    from their postprocess confidences: rotation, confidence bits, and every row of logits / ids / maps below the step
    count of the reading's pass (0 from there on where the steps shape the result), for R = 1, 2, 3, 4, orders other
    than ascending, allowlists, maps, refine_iters 0, NAR, ar_kernel 0 / 2, dec_depth 2, ViTSTR, host crops and crop
    counts that fill neither a reading group nor a super-chunk;
  * ties keep the first orientation; the threshold re-reads exactly the crops below it;
  * locate with orientations maps each crop back under its chosen rotation."""
import numpy as np
import pytest
import torch

import orientation_oracle as oo

pytestmark = pytest.mark.gpu


def _model(experiment, seed=0, **kw):
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config(experiment, **kw)
    m = create_model(experiment, **kw)
    m.model.load_state_dict(init_state_dict(cfg, seed))
    return m.eval().to("cuda")


@pytest.fixture(scope="module")
def parseq():
    return _model("parseq")


@pytest.fixture(scope="module")
def parseq_d2():
    return _model("parseq", seed=1, dec_depth=2)


@pytest.fixture(scope="module")
def vitstr():
    return _model("vitstr", img_size=(224, 224), patch_size=(16, 16))


def _crops(n, seed, cuda=True):
    rng = np.random.default_rng(seed)
    out = [torch.from_numpy(rng.integers(0, 256, (int(rng.integers(12, 70)), int(rng.integers(24, 220)), 3),
                                        dtype=np.uint8)) for _ in range(n)]
    return [c.cuda() for c in out] if cuda else out


def _restore(m):
    """Back to the default sizes (max_batch 512, chunk 512, dec_chunk 128) after a test shrank max_batch."""
    for k, v in (("max_batch", 256), ("dec_chunk", 128), ("max_batch", 512)):
        m.model.set_engine_option(k, v)


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    return torch.equal(_bits(a.cpu()), _bits(b.cpu()))


def _conf(m, logits):
    """parseq_postprocess's confidence of logits [N, L, C] (on the device)."""
    eng = m.model.engine()
    x = logits.cuda().contiguous()
    N, L, _ = x.shape
    ids = torch.empty((N, L), dtype=torch.int32, device="cuda")
    ln = torch.empty((N,), dtype=torch.int32, device="cuda")
    conf = torch.empty((N,), dtype=torch.float32, device="cuda")
    eng.postprocess(x.data_ptr(), N, L, ids.data_ptr(), ln.data_ptr(), conf.data_ptr(),
                    torch.cuda.current_stream().cuda_stream, 0)
    return conf.cpu()


def _launches(m, fn):
    eng = m.model.engine()
    torch.cuda.synchronize()
    before = eng.launches
    out = fn()
    torch.cuda.synchronize()
    return eng.launches - before, out


def _reading_steps(ids):
    """The AR step count each reading alone gives (kernels.cuh ar_steps_kernel): first EOS among positions 0..L-2,
    plus one, else L."""
    N, L = ids.shape
    out = []
    for row in ids.tolist():
        e = next((i for i, v in enumerate(row[:L - 1]) if v == 0), None)
        out.append(L if e is None else e + 1)
    return out


# ---------------------------------------------------------------- per-crop rotations
@pytest.mark.parametrize("where", ["cuda", "host", "small_max_batch"])
def test_rotation_list_reads_each_crop_at_its_rotation(parseq, where):
    m = parseq
    N = 10
    crops = _crops(N, 5, cuda=where != "host")
    rots = [0, 90, 180, 270, 90, 0, 270, 180, 180, 90]
    if where == "small_max_batch":
        m.model.set_engine_option("max_batch", 4)
    try:
        with torch.inference_mode():
            lg, ids, steps, maps = m.model._run(crops, None, True, 1, rotation=rots, attn_maps=True)
            uni = {r: m.model._run(crops, None, True, 1, rotation=r, attn_maps=True) for r in (0, 90, 180, 270)}
            single = [m.model._run([crops[b]], None, True, 1, rotation=rots[b])[2] for b in range(N)]
    finally:
        _restore(m)
    for b, r in enumerate(rots):
        assert _same(lg[b], uni[r][0][b]) and _same(ids[b], uni[r][1][b]) and _same(maps[b], uni[r][3][b]), (where, b)
    assert int(steps) == max(int(s) for s in single)
    assert lg.device.type == ("cpu" if where == "host" else "cuda")


def test_rotation_list_of_zeros_launches_as_rotation_0(parseq):
    crops = _crops(6, 6)
    with torch.inference_mode():
        m = parseq
        m.model._run(crops, None, True, 1, rotation=0)               # captures the graph
        n0, a = _launches(m, lambda: m.model._run(crops, None, True, 1, rotation=0))
        n1, b = _launches(m, lambda: m.model._run(crops, None, True, 1, rotation=[0] * 6))
    assert n0 == n1
    assert _same(a[0], b[0])


def test_rotation_list_in_preprocess_score_and_beam(parseq):
    crops = _crops(4, 7)
    rots = [270, 0, 90, 180]
    with torch.inference_mode():
        u8 = parseq.preprocess(crops, rots)
        for b, r in enumerate(rots):
            assert torch.equal(u8[b], parseq.preprocess([crops[b]], r)[0])
        assert torch.equal(parseq.score(crops, ["ab", "c"], rotation=rots), parseq.score(u8, ["ab", "c"]))
        la, sa = parseq.beam_search(crops, 3, rotation=rots)
        lb, sb = parseq.beam_search(u8, 3)
    assert la == lb and _same(sa, sb)


# ---------------------------------------------------------------- orientation search
def _expected(m, crops, orientations, t, decode_ar, refine, max_batch=512, mask=None, maps=False, vitstr=False):
    """The search assembled from the engine's own forward at each orientation and the fp64 rule."""
    runs = [m.model._run(crops, None, decode_ar, refine, rotation=r, class_mask=mask, attn_maps=maps)
            for r in orientations]
    conf = torch.stack([_conf(m, r[0]) for r in runs], 1)             # [N, R] fp32
    t32 = None if t is None else float(np.float32(t))
    pick, rr = oo.select(conf.double().numpy(), t32)
    N, L = runs[0][1].shape
    R1 = len(orientations) - 1
    zero_tail = decode_ar and refine == 0 and not vitstr
    s = [_reading_steps(r[1].cpu()) for r in runs]
    S1 = int(runs[0][2])
    S_pass = [S1] * N
    listed = [b for b in range(N) if rr[b]] if R1 else []
    steps = S1
    per = max_batch // R1 if R1 else 0
    for k0 in range(0, len(listed), max(per, 1)):
        chunk = listed[k0:k0 + per]
        Sc = max(s[r][b] for b in chunk for r in range(1, R1 + 1))
        steps = max(steps, Sc)
        for b in chunk:
            if pick[b] > 0:
                S_pass[b] = Sc
    out = {}
    for name, i in (("logits", 0), ("ids", 1), ("maps", 3)):
        if runs[0][i] is None:
            continue
        x = torch.stack([runs[pick[b]][i][b] for b in range(N)]).cpu().clone()
        if zero_tail:
            for b in range(N):
                x[b, S_pass[b]:] = 0
        out[name] = x
    out["rotation"] = torch.tensor([orientations[k] for k in pick])
    out["confidence"] = torch.stack([conf[b, pick[b]] for b in range(N)])
    out["rereads"] = len(listed)
    out["steps"] = steps if zero_tail else None
    out["one_chunk_steps"] = max(int(r[2]) for r in runs) if (R1 == 0 or len(listed) <= per) and t is None else None
    return out


def _check(m, crops, orientations, t=None, decode_ar=True, refine=1, max_batch=512, allowlist=None, maps=False,
           vitstr=False):
    N = len(crops)
    mask = m.allowlist_mask(allowlist, N)
    if max_batch != 512:
        m.model.set_engine_option("max_batch", max_batch)
    try:
        with torch.inference_mode():
            got = m.model._run_oriented(crops, orientations, t, None, decode_ar, refine, mask, maps)
            want = _expected(m, crops, orientations, t, decode_ar, refine, max_batch, mask, maps, vitstr)
            rereads = m.model.engine().debug_int("orient_rereads")
    finally:
        if max_batch != 512:
            _restore(m)
    logits, ids, steps, mp, rot, conf = got
    assert torch.equal(rot.cpu().long(), want["rotation"])
    assert _same(conf, want["confidence"])
    assert _same(logits, want["logits"])
    assert _same(ids, want["ids"])
    if maps:
        assert _same(mp, want["maps"])
    if want["steps"] is not None:
        assert int(steps) == want["steps"]
    if want["one_chunk_steps"] is not None:
        assert int(steps) == want["one_chunk_steps"]
    assert rereads == want["rereads"]
    # the returned confidence is postprocess's of the returned logits
    assert _same(_conf(m, logits), conf)
    return got, want


@pytest.mark.parametrize("orientations", [(0, 90, 180, 270), (0, 180), (270, 0, 90), (180,), (90, 270, 0, 180)])
def test_search_equals_per_rotation_forwards(parseq, orientations):
    _check(parseq, _crops(13, 11), orientations)


@pytest.mark.parametrize("case", ["allowlist_maps", "refine0_tail", "nar", "ar_kernel0", "host", "uneven_chunks"])
def test_search_schedules(parseq, case):
    m, crops = parseq, _crops(11, 12, cuda=case != "host")
    if case == "allowlist_maps":
        _check(m, crops, (0, 90, 180, 270), allowlist=["0123456789", None, "abc", ""] + [None] * 7, maps=True)
    elif case == "refine0_tail":
        _check(m, crops, (90, 0, 270), refine=0, maps=True)
    elif case == "nar":
        _check(m, crops, (0, 180), decode_ar=False, refine=2)
    elif case == "ar_kernel0":
        m.model.set_engine_option("ar_kernel", 0)
        try:
            _check(m, crops, (0, 90, 180, 270), refine=0)
        finally:
            m.model.set_engine_option("ar_kernel", 2)
    elif case == "host":
        got, _ = _check(m, crops, (0, 90, 180, 270), refine=0)
        assert got[0].device.type == "cpu"
    else:
        # super-chunks of 7 // 3 = 2 crops: 6 readings, rounded to 7 (max_batch); 11 crops -> 6 super-chunks
        _check(m, crops, (0, 90, 180, 270), refine=0, max_batch=7)
        _check(m, crops, (0, 90, 180, 270), max_batch=7, allowlist="0123456789abcdef")
        # host crops staged per super-chunk: pass 1 in two, pass 2 in six packed super-chunks
        _check(m, _crops(11, 12, cuda=False), (0, 90, 180, 270), refine=0, max_batch=7)


def test_search_dec_depth_2(parseq_d2):
    _check(parseq_d2, _crops(9, 13), (0, 90, 180, 270), maps=True)
    _check(parseq_d2, _crops(9, 13), (180, 0), refine=0)


def test_search_vitstr(vitstr):
    _check(vitstr, _crops(9, 14), (0, 90, 180, 270), decode_ar=False, refine=0, vitstr=True)
    _check(vitstr, _crops(9, 14), (270, 90), t=0.5, decode_ar=False, refine=0, vitstr=True)


def test_ties_keep_the_first_orientation(parseq):
    """A constant-colour crop resizes to the same image in every orientation, so its readings tie."""
    crops = [torch.full((h, w, 3), v, dtype=torch.uint8, device="cuda") for h, w, v in ((20, 60, 128), (50, 17, 3),
                                                                                        (31, 31, 250))]
    got, _ = _check(parseq, crops, (90, 0, 180, 270))
    assert got[4].tolist() == [90, 90, 90]


def test_threshold(parseq):
    m = parseq
    crops = _crops(16, 15)
    full, _ = _check(m, crops, (0, 90, 180, 270))
    with torch.inference_mode():
        m.model.engine().set_option("timing", 1)
        try:
            zero, _ = _check(m, crops, (0, 90, 180, 270), t=0.0)
            torch.cuda.synchronize()
            t0 = m.model.engine().get_timing()["orient"]["launches"]
        finally:
            m.model.engine().set_option("timing", 0)
        base = m.model._run(crops, None, True, 1, rotation=0)
    assert t0 == 1                                                    # the confidence kernel, no pass 2
    assert _same(zero[0], base[0]) and (zero[4] == 0).all()
    above, _ = _check(m, crops, (0, 90, 180, 270), t=1.5)
    for a, b in zip(above, full):
        assert (a is None and b is None) or _same(a, b)
    c0 = _conf(m, base[0])
    t = float(torch.sort(c0).values[8])                              # half the crops below t
    m.model.set_engine_option("max_batch", 6)
    try:
        with torch.inference_mode():
            eng = m.model.engine()
            eng.set_option("timing", 1)
            m.model._run_oriented(crops, (0, 90, 180, 270), t, None, True, 1)
            torch.cuda.synchronize()
            sel = eng.get_timing()["orient"]["launches"]
            eng.set_option("timing", 0)
            rereads, readings = eng.debug_int("orient_rereads"), eng.debug_int("orient_readings")
    finally:
        _restore(m)
    listed = int((c0 < np.float32(t)).sum())
    assert rereads == listed and 0 < listed < len(crops)
    assert sel == 1 + 2 * ((listed + 1) // 2)            # init, then confidence + select per super-chunk of 2 crops
    assert readings == 6 * (listed // 2) + (4 if listed % 2 else 0)
    _check(m, crops, (0, 90, 180, 270), t=t, max_batch=6)


def test_locate_with_orientations(parseq):
    crops = _crops(6, 16)
    with torch.inference_mode():
        _, rot, _ = parseq.read_oriented(crops, (0, 90, 180, 270))
        labels, confs, centers, boxes = parseq.locate(crops, orientations=(0, 90, 180, 270))
        for b, r in enumerate(rot.tolist()):
            lb, cb, ce, bx = parseq.locate([crops[b]], rotation=r)
            assert labels[b] == lb[0] and confs[b] == cb[0]
            assert torch.equal(centers[b], ce[0]) and torch.equal(boxes[b], bx[0])


# ---------------------------------------------------------------- against the reference's own modules
@pytest.mark.parametrize("case", ["or_s_sharp", "or_ti_c3001", "or_vitstr_s"])
def test_choice_and_ids_match_the_reference_goldens(case):
    """tests/golden/orientation (tests/make_golden_orientation.py): the reference's fp64 reading of every golden crop in
    every orientation and the orientation the rule picks by its `_eval_step` confidence.  On crops whose best and
    second-best confidences differ by more than 5 % and whose every greedy decision, in every orientation, clears a
    2e-2 margin, the engine chooses the same orientation and reads the same ids through the EOS."""
    import os
    import make_golden_orientation as mg
    from make_golden_long import charset
    from parseq_b200.factory import create_model
    from parseq_b200.weights import state_dict_digest
    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "orientation", case + ".pt"),
                   weights_only=False)
    cfg = mg.case_config(g["experiment"], g["n_extra"])
    sd = mg.state_dict(cfg, g["weight_seed"], g["sharp"])
    assert state_dict_digest(sd) == g["sd_digest"]
    m = create_model(g["experiment"], charset_train=charset(g["n_extra"]), max_label_length=cfg.max_label_length)
    (m if g["experiment"] == "vitstr" else m.model).load_state_dict(sd)
    m = m.eval().to("cuda")
    crops = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in mg.crops()]
    vitstr = g["experiment"] == "vitstr"
    with torch.inference_mode():
        _, ids, _, _, rot, _ = m.model._run_oriented(crops, g["orientations"], None, None, False if vitstr else cfg.decode_ar,
                                                     0 if vitstr else cfg.refine_iters)
    conf = g["confidence"].T                                           # [N, R]
    top = conf.sort(dim=1, descending=True).values
    clear = ((top[:, 0] - top[:, 1]) > 0.05 * top[:, 0]) & (g["min_margin"].min(0).values > 2e-2)
    L = ids.shape[1]
    full = torch.tensor([s == L for s in g["steps"]])
    clear &= ((g["length"] < torch.tensor(g["steps"])[:, None]) | full[:, None]).all(0)
    assert int(clear.sum()) >= 3, (case, int(clear.sum()))
    ids, rot = ids.cpu(), rot.cpu()
    for b in torch.nonzero(clear).flatten().tolist():
        k = int(g["chosen"][b])
        assert int(rot[b]) == g["orientations"][k], (case, b)
        n = int(g["length"][k, b])
        want = g["ids"][k, b, :n + 1].long()
        assert torch.equal(ids[b, :want.numel()].long(), want), (case, b)
