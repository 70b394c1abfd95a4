"""GPU: cross-attention maps (parseq_forward_args.attn_maps, PARSeq.read_with_attention / locate).

  * The maps of every schedule (AR without refinement, NAR, AR + refinement, NAR + 2 refinements) against the fp64
    rounding-point maps of tests/attn_maps_reference.py fed the engine's own bf16 memory and the engine's own ids, within
    attn_maps_reference.BOUNDS, at depth 1 and 2, T = 128 / 196 / 256 and L = 26 / 64.
  * Asking for maps changes nothing else: for every schedule and entry point (float, uint8, crops and their host
    variants), with the CUDA graphs and eagerly (timing mode), the logits, ids and steps are byte-identical with and
    without maps, and a call without maps launches the kernels the parent commit launched (PARENT_LAUNCHES).
  * The maps are bitwise the same whichever AR loop ran (where the ids agree) and whatever batch an image is in.
  * locate on raw crops agrees with locate on the preprocessed crops mapped back; ViTSTR and teacher forcing are
    rejected with the documented errors."""
import functools
import os

import pytest
import torch

from attn_maps_reference import BOUNDS, GOLDEN_BOUNDS, MapsReference, excess, format_stats, map_stats
from token_count_geometries import geometry_config

pytestmark = pytest.mark.gpu

SCHEDULES = {"ar": (True, 0), "nar": (False, 0), "ar_refine": (True, 1), "nar_refine2": (False, 2)}


@functools.lru_cache(maxsize=4)
def _model(exp="parseq", T=None, mll=25, depth=1, sharp=4.0, fuse_ln0=True):
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    over = dict(geometry_config(T, exp)[1]) if T is not None else dict(enc_depth=2)
    over.update(max_label_length=mll, dec_depth=depth)
    cfg = make_config(exp, **over)
    sd = init_state_dict(cfg, 5, sharp=sharp)
    m = create_model(exp, **over)
    m.model.load_state_dict(sd)
    m = m.eval().to("cuda")
    if fuse_ln0:
        m.model.set_engine_option("fuse_ln", 0)     # encode() returns the memory forward's decoder reads
    return cfg, sd, m


def _images(cfg, B, seed):
    from parseq_b200.weights import synth_images
    return synth_images(cfg, B, seed).cuda()


def _run(m, x, sched, maps=True, max_length=None, class_mask=None):
    ar, refine = SCHEDULES[sched]
    m.model.decode_ar, m.model.refine_iters = ar, refine
    with torch.inference_mode():
        return m.model._run(x, max_length, ar, refine, class_mask=class_mask, attn_maps=maps)


def _assert_distributions(maps):
    assert bool((maps >= 0).all())
    assert float((maps.double().sum(-1) - 1).abs().max()) <= 1e-5


# ---- against the fp64 rounding-point maps --------------------------------------------------------------------------
BOUND_CASES = [("parseq", None, 25, 1), ("parseq", None, 25, 2), ("parseq-patch16-224", None, 25, 1),
               ("parseq", 256, 25, 1), ("parseq", None, 63, 1), ("parseq-tiny", None, 25, 1)]


@pytest.mark.parametrize("sched", sorted(SCHEDULES))
@pytest.mark.parametrize("case", BOUND_CASES, ids=[f"{e}-T{t}-mll{m}-d{d}" for e, t, m, d in BOUND_CASES])
def test_maps_within_rounding_point_bound(case, sched):
    exp, T, mll, depth = case
    cfg, sd, m = _model(exp, T, mll, depth)
    B, L = 6, mll + 1
    x = _images(cfg, B, 40)
    with torch.inference_mode():
        mem = m.model.encode(x)
    _, ids, _, maps = _run(m, x, sched, max_length=mll)
    _assert_distributions(maps)
    ref = MapsReference(cfg, sd, device="cuda")
    bos = cfg.num_tokens - 2

    def ctx(sched0):
        prev = _run(m, x, sched0, maps=False, max_length=mll)[1]
        return torch.cat([torch.full((B, 1), bos, dtype=torch.long, device=prev.device), prev[:, :L - 1].long()], 1)

    if sched == "ar":
        want = ref.ar(mem, ids)
    elif sched == "nar":
        want = ref.nar(mem, L)
    elif sched == "ar_refine":
        want = ref.refine(mem, [ctx("ar")])
    else:
        m.model.refine_iters = 1
        with torch.inference_mode():
            ids1 = m.model._run(x, mll, False, 1)[1]
        c2 = torch.cat([torch.full((B, 1), bos, dtype=torch.long, device=ids1.device), ids1[:, :L - 1].long()], 1)
        want = ref.refine(mem, [ctx("nar"), c2])
    assert maps.shape == want.shape == (B, L, cfg.num_patches)
    s = map_stats(maps, want)
    print(format_stats(f"[{exp} T{cfg.num_patches} mll{mll} depth{depth} {sched}]", s))
    assert max(excess(s).values()) <= 1.0, (s, BOUNDS)


# ---- against the reference's own maps (tests/golden/attention, tests/make_golden_attention.py) ------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "attention")
GOLDENS = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.endswith(".pt")) if os.path.isdir(GOLDEN) else []
MARGIN = 2e-2      # an image's ids are the reference's where every greedy decision clears the engine's bf16 error


@pytest.mark.parametrize("name", GOLDENS)
def test_goldens(name):
    from make_golden_attention import golden_state_dict
    from make_golden_long import make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import state_dict_digest, synth_images
    blob = torch.load(os.path.join(GOLDEN, name + ".pt"))
    exp, mll, B = blob["experiment"], blob["max_label_length"], blob["batch"]
    img = (224, 224) if exp == "parseq-patch16-224" else (32, 128)
    cfg = make_config_long(exp, mll, blob["n_extra"], img_size=img, dec_depth=blob["dec_depth"])
    sd = golden_state_dict(cfg, blob["weight_seed"], blob["sharp"], blob["eos_bias"])
    assert state_dict_digest(sd) == blob["sd_digest"]
    m = create_model(exp, charset_train=cfg.charset_train, max_label_length=mll, img_size=img,
                     dec_depth=blob["dec_depth"], decode_ar=blob["decode_ar"], refine_iters=blob["refine_iters"])
    m.model.load_state_dict(sd)
    m = m.eval().to("cuda")
    x = synth_images(cfg, B, blob["image_seed"]).cuda()
    mask = m.allowlist_mask(blob["allowlist"], B) if blob["allowlist"] is not None else None
    with torch.inference_mode():
        logits, ids, maps = m.model.forward_with_attention(x, blob["max_length"], class_mask=mask)
    _assert_distributions(maps)
    clear = (blob["min_margin"] > MARGIN).tolist()
    assert any(clear), name
    if all(clear):
        assert maps.shape == blob["maps"].shape, (maps.shape, blob["maps"].shape)
    got, want = [], []
    for b in range(B):
        if not clear[b]:
            continue
        ref_ids = blob["ids"][b].long()
        eos = (ref_ids == 0).nonzero()
        n = int(eos[0]) if len(eos) else ref_ids.numel() - 1          # the label's rows: up to its EOS
        assert torch.equal(ids[b, :n + 1].cpu().long(), ref_ids[:n + 1]), (name, b)
        got.append(maps[b, :n + 1])
        want.append(blob["maps"][b, :n + 1])
    s = map_stats(torch.cat(got), torch.cat(want))
    print(format_stats(f"[{name}]", s))
    assert all(s[k] <= v for k, v in GOLDEN_BOUNDS.items()), (name, s, GOLDEN_BOUNDS)


# ---- nothing else changes -----------------------------------------------------------------------------------------
ENTRIES = ("float", "u8", "crops", "host_float", "host_u8", "host_crops")
# parseq_kernel_launches of one call without maps (PARSeq-S with a depth-2 encoder and the engine's default options, 3
# images, max_length None), as the
# parent commit launches them, measured with its library through call_entry: the float and uint8 entry points and their
# host variants, with the CUDA graph and eagerly alike; the raw-crop entry points add the resize kernel
_PARENT_BASE = {"ar": 21, "ar_refine": 34, "nar": 30, "nar_refine2": 56}
PARENT_LAUNCHES = {s: {mode: {e: n + (1 if e.endswith("crops") else 0) for e in ("float", "u8", "crops", "host_float",
                                                                                  "host_u8", "host_crops")}
                       for mode in ("graph", "eager")} for s, n in _PARENT_BASE.items()}


def _inputs(cfg, B):
    from parseq_b200.system import pack_crops
    g = torch.Generator().manual_seed(3)
    crops = [torch.randint(0, 256, (int(h), int(w), 3), generator=g, dtype=torch.uint8)
             for h, w in [(40, 150), (20, 90), (64, 64)][:B]]
    H, W = cfg.img_size
    u8 = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    x = u8.permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5).contiguous()
    return {"float": x.cuda(), "u8": u8.cuda(), "crops": pack_crops([c.cuda() for c in crops]),
            "host_float": x.pin_memory(), "host_u8": u8.pin_memory(), "host_crops": pack_crops(crops, pin_memory=True)}


def call_entry(m, entry, inp, B, sched, maps):
    """One engine call through `entry`: (logits, ids, steps, maps or None, kernel launches of the call)."""
    from parseq_b200.system import _crops_c
    eng = m.model.engine()
    cfg = m.model.cfg
    ar, refine = SCHEDULES[sched]
    host = entry.startswith("host")
    dev = torch.device("cpu") if host else torch.device("cuda")
    L = eng.num_steps(None)
    logits = torch.empty((B, L, cfg.num_classes), dtype=torch.float32, device=dev, pin_memory=host)
    ids = torch.empty((B, L), dtype=torch.int32, device=dev, pin_memory=host)
    steps = torch.empty((1,), dtype=torch.int32, device=dev, pin_memory=host)
    amap = torch.empty((B, L, cfg.num_patches), dtype=torch.float32, device=dev, pin_memory=host) if maps else None
    mp = amap.data_ptr() if maps else None
    st = torch.cuda.current_stream().cuda_stream
    before = eng.launches
    ptrs = (logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), st, None, ar, refine)
    kw = {"attn_maps_ptr": mp} if maps else {}
    if entry in ("float", "host_float"):
        fn = eng.forward if entry == "float" else eng.forward_host
        fn(inp.data_ptr(), B, *ptrs, **kw)
    elif entry in ("u8", "host_u8"):
        eng.forward_u8(inp.data_ptr(), B, *ptrs, host=host, **kw)
    else:
        data, offsets, sizes = inp
        eng.forward_crops(_crops_c(data, offsets, sizes, 0), B, *ptrs, host=host, **kw)
    torch.cuda.synchronize()
    return logits, ids, steps, amap, eng.launches - before


@pytest.mark.parametrize("mode", ("graph", "eager"))
@pytest.mark.parametrize("sched", sorted(SCHEDULES))
def test_maps_change_nothing_else(sched, mode):
    cfg, sd, m = _model(fuse_ln0=False)               # the engine's default options
    B = 3
    inputs = _inputs(cfg, B)
    eng = m.model.engine()
    eng.set_option("timing", 1 if mode == "eager" else 0)
    try:
        for entry in ENTRIES:
            base = call_entry(m, entry, inputs[entry], B, sched, False)
            got = call_entry(m, entry, inputs[entry], B, sched, True)
            again = call_entry(m, entry, inputs[entry], B, sched, False)
            for k in range(3):
                assert torch.equal(base[k].view(torch.int32), got[k].view(torch.int32)), (entry, k)
                assert torch.equal(base[k].view(torch.int32), again[k].view(torch.int32)), (entry, k)
            _assert_distributions(got[3])
            assert base[4] == again[4] == PARENT_LAUNCHES[sched][mode][entry], (entry, base[4], again[4])
    finally:
        eng.set_option("timing", 0)


# ---- bitwise reproducibility --------------------------------------------------------------------------------------
def test_ar_maps_do_not_depend_on_the_ar_loop():
    cfg, sd, m = _model()
    x = _images(cfg, 24, 50)
    res = {}
    for k in (0, 1, 2):
        m.model.set_engine_option("ar_kernel", k)
        _, ids, _, maps = _run(m, x, "ar", max_length=25)
        res[k] = (ids, maps, m.model.engine().debug_int("ar_last_path"))
    m.model.set_engine_option("ar_kernel", 2)
    assert [res[k][2] for k in (0, 1, 2)] == [0, 1, 2]
    for k in (0, 1):
        same = (res[k][0] == res[2][0]).all(dim=1)
        assert int(same.sum()) >= 12, int(same.sum())
        assert torch.equal(res[k][1][same], res[2][1][same]), k


@pytest.mark.parametrize("sched", sorted(SCHEDULES))
def test_maps_do_not_depend_on_the_batch(sched):
    cfg, sd, m = _model()
    x = _images(cfg, 150, 60)
    eng = m.model.engine()
    whole = _run(m, x, sched, max_length=25)[3]
    one = _run(m, x[:1], sched, max_length=25)[3]
    seven = _run(m, x[:7], sched, max_length=25)[3]
    try:
        eng.set_option("max_batch", 64)           # three super-chunks ...
        eng.set_option("dec_chunk", 16)           # ... of four decoder groups
        split = _run(m, x, sched, max_length=25)[3]
    finally:
        eng.set_option("max_batch", 512)
        eng.set_option("dec_chunk", 128)
    _assert_distributions(whole)
    assert torch.equal(one[0], whole[0])
    assert torch.equal(seven, whole[:7])
    assert torch.equal(split, whole)


def test_read_with_attention_shapes_and_allowlist():
    cfg, sd, m = _model()
    x = _images(cfg, 4, 70)
    for sched in SCHEDULES:
        m.model.decode_ar, m.model.refine_iters = SCHEDULES[sched]
        with torch.inference_mode():
            ref = m(x)
            logits, maps = m.read_with_attention(x)
            allow_logits, allow_maps = m.read_with_attention(x, allowlist="0123456789")
            plain = m(x, allowlist="0123456789")
        assert torch.equal(logits, ref) and torch.equal(allow_logits, plain)
        gh, gw = cfg.grid
        assert maps.shape == (4, logits.shape[1], gh, gw) and allow_maps.shape[1] == allow_logits.shape[1]
        _assert_distributions(allow_maps.flatten(2))


# ---- locate ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rotation", (0, 90, 180, 270))
def test_locate_on_crops_agrees_with_preprocessed(rotation):
    from parseq_b200.system import unrotate_boxes, unrotate_points
    cfg, sd, m = _model()
    m.model.decode_ar, m.model.refine_iters = True, 1
    g = torch.Generator().manual_seed(rotation)
    crops = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8) for h, w in [(40, 150), (90, 30), (33, 33)]]
    with torch.inference_mode():
        labels, confs, centers, boxes = m.locate(crops, rotation=rotation)
        pre = m.preprocess(crops, rotation)
        labels2, confs2, centers2, boxes2 = m.locate(pre)
    assert labels == labels2 and confs == confs2
    for b, c in enumerate(crops):
        hw = tuple(c.shape[:2])
        assert centers[b].shape == (len(labels[b]), 2) and boxes[b].shape == (len(labels[b]), 4)
        back = unrotate_points(centers2[b].cpu(), hw, cfg.img_size, rotation)
        assert torch.allclose(centers[b].cpu(), back, rtol=0, atol=1e-3), b
        assert torch.allclose(boxes[b].cpu(), unrotate_boxes(boxes2[b].cpu(), hw, cfg.img_size, rotation), rtol=0, atol=1e-3)


# ---- rejections -----------------------------------------------------------------------------------------------------
def test_vitstr_and_teacher_forcing_are_rejected():
    from parseq_b200.engine import EngineError
    from parseq_b200.factory import create_model
    cfg, sd, m = _model()
    x = _images(cfg, 2, 80)
    eng = m.model.engine()
    L = eng.num_steps(None)
    logits = torch.empty((2, L, cfg.num_classes), device="cuda")
    maps = torch.empty((2, L, cfg.num_patches), device="cuda")
    forced = torch.zeros((2, L), dtype=torch.int32, device="cuda")
    with pytest.raises(EngineError, match="error -1"):
        eng.forward(x.data_ptr(), 2, logits.data_ptr(), None, None, torch.cuda.current_stream().cuda_stream,
                    forced_ids_ptr=forced.data_ptr(), attn_maps_ptr=maps.data_ptr())
    with pytest.raises(ValueError):
        m.model._run(x, None, True, 1, forced_ids=forced, attn_maps=True)
    v = create_model("vitstr", enc_depth=2).eval().to("cuda")
    vx = _images(v.model.cfg, 2, 81)
    ve = v.model.engine()
    vl = torch.empty((2, L, v.model.cfg.num_classes), device="cuda")
    with pytest.raises(EngineError, match="error -2"):
        ve.forward(vx.data_ptr(), 2, vl.data_ptr(), None, None, torch.cuda.current_stream().cuda_stream,
                   decode_ar=False, refine_iters=0, attn_maps_ptr=maps.data_ptr())
    with pytest.raises(NotImplementedError):
        v.read_with_attention(vx)
    with pytest.raises(NotImplementedError):
        v.locate(vx)
