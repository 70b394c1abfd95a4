"""Curved text regions on the GPU (parseq_warp_polygons, region_tps_kernel, crop_regions with polygons):
  * the kernel's bytes equal the fp64 restatement (tps_warp_oracle.py) on every golden polygon away from fragile pixels
    (those whose byte changes under a 1e-7 px move of the mapped point), through crop_regions and through the C ABI
    with more regions than max_batch and ragged k in one call;
  * an affine polygon gives the crop of its quad; a call mixing quads and polygons gives the bytes of the quads-only
    and polygons-only calls without a copy; CPU and PIL frames give the bytes of CUDA frames;
  * model calls on the crops equal those on cloned separate crops (PARSeq-S, PARSeq-Ti, ViTSTR), and read_oriented,
    score, beam_search and locate take them;
  * to_frame sends crop corners to the polygon's corners; the table's device memory goes with the handle."""
import numpy as np
import pytest
import torch

import make_golden_curved as mgc
from parseq_b200.regions import engine_points
from tps_warp_oracle import fragile, warp

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
def golden():
    frames, g = mgc.load()
    expect = []
    for p, f, (h, w) in zip(g["polygons"], g["frame_index"], g["sizes"]):
        from parseq_b200.engine import tps_coeffs
        t = tps_coeffs(engine_points(p.tolist()))
        expect.append((warp(frames[f], h, w, t), fragile(frames[f], h, w, t)))
    return frames, g, expect


def _check(crops, g, expect, label):
    """Zero mismatches away from fragile pixels on every case.  The fragile share is below 1e-4 over all cases and in
    every case but one, the 220-degree k = 32 sector (6 of its 5 380 pixels, 1.1e-3); the bound per case is 2e-3."""
    fragile_px, pixels = 0, 0
    for i, (c, (want, frag)) in enumerate(zip(crops, expect)):
        got = c.cpu().numpy() if isinstance(c, torch.Tensor) else c
        assert got.shape == want.shape, (label, i)
        bad = (got != want).any(-1) & ~frag
        assert not bad.any(), f"{label}: region {i} differs at {int(bad.sum())} non-fragile pixels"
        differ = int(((got != want).any(-1) & frag).sum())
        if frag.any():
            print(f"{label}: region {i} {frag.shape}: {int(frag.sum())} fragile pixels ({frag.mean():.2e}), "
                  f"{differ} of them differ")
        assert frag.mean() < 2e-3, (label, i, float(frag.mean()))
        fragile_px, pixels = fragile_px + int(frag.sum()), pixels + frag.size
    print(f"{label}: fragile share over all cases {fragile_px / pixels:.2e}")
    assert fragile_px / pixels < 1e-4


def test_kernel_equals_oracle_on_goldens(parseq, golden):
    frames, g, expect = golden
    with torch.inference_mode():
        rc = parseq.crop_regions([torch.from_numpy(f).cuda() for f in frames], g["polygons"],
                                 frame_index=g["frame_index"])
    assert [tuple(c.shape[:2]) for c in rc] == [tuple(s) for s in g["sizes"]]
    _check(rc, g, expect, "crop_regions")


def test_c_abi_past_max_batch_with_ragged_k(golden):
    from parseq_b200.engine import PolygonsC
    frames, g, expect = golden
    m = _model("parseq-tiny")
    m.model.set_engine_option("max_batch", 8)                 # 30 regions: four chunks, the last one partial
    eng = m.model.engine()
    fdata = torch.cat([torch.from_numpy(f).reshape(-1) for f in frames]).cuda()
    nb = [3 * f.shape[0] * f.shape[1] for f in frames]
    fo = np.concatenate([[0], np.cumsum(nb)[:-1]]).astype(np.int64)
    fs = np.array([f.shape[:2] for f in frames], dtype=np.int32)
    fi = np.array(g["frame_index"], dtype=np.int32)
    sz = np.array(g["sizes"], dtype=np.int32)
    pts = [engine_points(p.tolist()) for p in g["polygons"]]
    npt = np.array([len(p) for p in pts], dtype=np.int32)
    assert len(set(npt.tolist())) > 3
    flat = np.array([xy for p in pts for xy in p], dtype=np.float64)
    total = int((3 * sz[:, 0].astype(np.int64) * sz[:, 1]).sum())
    out = torch.empty(total, dtype=torch.uint8, device="cuda")
    pc = PolygonsC(fdata.data_ptr(), fdata.numel(), fo.ctypes.data, fs.ctypes.data, len(frames), fi.ctypes.data,
                   sz.ctypes.data, npt.ctypes.data, flat.ctypes.data)
    eng.warp_polygons(pc, len(pts), out.data_ptr(), total, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    crops, o = [], 0
    for h, w in sz.tolist():
        crops.append(out[o:o + 3 * h * w].view(h, w, 3))
        o += 3 * h * w
    _check(crops, g, expect, "C ABI, max_batch 8")


def test_affine_polygon_equals_its_quad(parseq, golden):
    frames, _, _ = golden
    fr = torch.from_numpy(frames[0]).cuda()
    for cx, cy, w, h, a, k in ((160.3, 120.7, 140, 32, 0.4, 7), (200.0, 110.0, 90, 24, -1.1, 16), (100.0, 90.0, 60, 20, 2.5, 3)):
        p = mgc.affine_polygon(cx, cy, w, h, a, k)
        kk = len(p) // 2
        quad = [p[0], p[kk - 1], p[kk], p[-1]]
        with torch.inference_mode():
            a_ = parseq.crop_regions(fr, [p])[0].cpu().numpy()
            b_ = parseq.crop_regions(fr, [quad])[0].cpu().numpy()
        from parseq_b200.engine import tps_coeffs
        frag = fragile(frames[0], *a_.shape[:2], tps_coeffs(engine_points(p)))
        assert a_.shape == b_.shape
        assert not ((a_ != b_).any(-1) & ~frag).any(), (cx, cy, k)


def test_mixed_call_equals_separate_calls_without_a_copy(parseq, golden):
    from parseq_b200.system import pack_crops
    frames, g, _ = golden
    fr = [torch.from_numpy(f).cuda() for f in frames[:2]]
    quads = [[(10.0, 20.0), (120.0, 25.0), (118.0, 50.0), (12.0, 45.0)], [(200.0, 100.0), (300.0, 90.0), (305.0, 130.0), (198.0, 128.0)]]
    polys = [p for p, f in zip(g["polygons"], g["frame_index"]) if f < 2][:5]
    pf = [f for f in g["frame_index"] if f < 2][:5]
    regions = [polys[0].numpy(), np.array(quads[0]), polys[1].numpy(), polys[2].numpy(), np.array(quads[1]), polys[3].numpy(), polys[4].numpy()]
    kinds = ["p", "q", "p", "p", "q", "p", "p"]
    index = [pf[0], 0, pf[1], pf[2], 1, pf[3], pf[4]]
    with torch.inference_mode():
        mixed = parseq.crop_regions(fr, regions, frame_index=index)
        q_only = parseq.crop_regions(fr, quads, frame_index=[0, 1])
        p_only = parseq.crop_regions(fr, [p for p in polys], frame_index=pf)
    qs, ps = iter(q_only), iter(p_only)
    for kind, c in zip(kinds, mixed):
        assert torch.equal(c, next(qs) if kind == "q" else next(ps))
    qbytes = sum(c.numel() for c in q_only)
    assert mixed.offsets.tolist()[1] == 0 and mixed.offsets.tolist()[4] == q_only[0].numel()
    assert mixed.offsets.tolist()[0] == qbytes
    d, o, s = pack_crops(mixed)
    assert d is mixed.data and o is mixed.offsets
    assert all(c.data_ptr() >= d.data_ptr() and c.data_ptr() < d.data_ptr() + d.numel() for c in mixed)
    assert [p is None for p in mixed.polygons] == [k == "q" for k in kinds]
    assert all(torch.isnan(mixed.coeffs[i]).all() == (k == "p") for i, k in enumerate(kinds))
    with torch.inference_mode():
        sep = [c.clone() for c in mixed]
        assert _eq(parseq(mixed), parseq(sep))          # non-monotone offsets through the crop entry points


def test_cpu_and_pil_frames_equal_cuda_frames(parseq, golden):
    from PIL import Image
    frames, g, _ = golden
    keep = [i for i, f in enumerate(g["frame_index"]) if f != 3]
    fr = frames[:3] + frames[4:]
    index = [{0: 0, 1: 1, 2: 2, 4: 3}[g["frame_index"][i]] for i in keep]
    polys = [g["polygons"][i] for i in keep]
    with torch.inference_mode():
        ref = parseq.crop_regions([torch.from_numpy(f).cuda() for f in fr], polys, frame_index=index)
        cpu = parseq.crop_regions([torch.from_numpy(f) for f in fr], polys, frame_index=index)
        pil = parseq.crop_regions([Image.fromarray(f) for f in fr], [p.numpy() for p in polys], frame_index=np.array(index))
    for a, b, c in zip(ref, cpu, pil):
        assert torch.equal(a, b) and torch.equal(a, c)


def _workload(n, seed, shape=(480, 640)):
    """Seeded curved words (arcs of k = 3..16 points) of two blocky frames."""
    import make_golden_regions as mg
    rng = np.random.default_rng(seed)
    H, W = shape
    frames = [torch.from_numpy(mg.make_frame(H, W, seed + k, 4)).cuda() for k in range(2)]
    polys, index = [], []
    while len(polys) < n:
        k = int(rng.choice([3, 5, 7, 16]))
        r, a0, span = rng.uniform(60, 400), rng.uniform(-150, -30), rng.uniform(10, 60) * rng.choice([-1, 1])
        p = mgc.band(mgc.arc(rng.uniform(0, W), rng.uniform(0, H) + r, r, a0 - span / 2, a0 + span / 2), k, rng.uniform(8, 30))
        try:
            from parseq_b200.regions import check_polygon
            check_polygon(p)
        except ValueError:
            continue
        polys.append(np.array(p))
        index.append(len(polys) % 2)
    return frames, polys, index


def _eq(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_eq(x, y) for x, y in zip(a, b))
    return a == b


@pytest.fixture(scope="module")
def regions(parseq):
    frames, polys, index = _workload(40, 9)
    with torch.inference_mode():
        rc = parseq.crop_regions(frames, polys, frame_index=index)
    return rc, [c.clone() for c in rc]


@pytest.mark.parametrize("name, kw", [("parseq", {}), ("parseq-tiny", {"refine_iters": 0}),
                                      ("vitstr", {"img_size": (224, 224), "patch_size": (16, 16)})])
def test_model_on_polygon_crops_equals_separate_crops(parseq, regions, name, kw):
    m = parseq if name == "parseq" else _model(name, **kw)
    rc, sep = regions
    with torch.inference_mode():
        assert _eq(m(rc), m(sep))


def test_read_oriented_score_beam_and_locate_on_polygon_crops(parseq, regions):
    rc, sep = regions
    words = ["text", "word", "hello", "a", "region"]
    with torch.inference_mode():
        assert _eq(parseq.read_oriented(rc, min_confidence=0.5), parseq.read_oriented(sep, min_confidence=0.5))
        assert _eq(parseq.score(rc, words), parseq.score(sep, words))
        assert _eq(parseq.beam_search(rc, 3), parseq.beam_search(sep, 3))
        assert _eq(parseq.locate(rc), parseq.locate(sep))
        _, _, centers, _ = parseq.locate(rc)
    for i, c in enumerate(centers):
        if len(c):
            p = rc.to_frame(c.double().cpu(), i)
            assert bool(torch.isfinite(p).all())


def test_to_frame_sends_crop_corners_to_polygon_corners(regions):
    """The corners are fiducials; GridGenerator's phi = r^2 ln(r + 1e-6) against the solve's r^2 ln r moves them by
    micro-pixels, so they are held to 1e-4 px (and within 1e-9 px where the spline is affine)."""
    rc, _ = regions
    for i, c in enumerate(rc):
        h, w = c.shape[:2]
        corners = rc.to_frame(torch.tensor([[0.0, 0.0], [w, 0.0], [w, h], [0.0, h]]), i)
        assert float((corners - rc.quads[i]).abs().max()) <= 1e-4, i
        p = rc.polygons[i]
        k = len(p) // 2
        assert torch.equal(rc.quads[i], torch.stack([p[0], p[k - 1], p[k], p[-1]]))


def test_table_memory_goes_with_the_handle():
    import gc
    from parseq_b200.engine import load_library
    lib = load_library()

    def live():
        gc.collect()
        torch.cuda.synchronize()
        return int(lib.parseq_debug_int(None, b"live_device_bytes"))
    frames, polys, index = _workload(5, 3)
    before = live()
    m = _model("parseq-tiny")
    with torch.inference_mode():
        m.crop_regions(frames, polys[:1], frame_index=index[:1])
        one = live()
        rc = m.crop_regions(frames, polys, frame_index=index)
    del rc
    assert live() == one                   # the table is allocated once, at max_batch regions
    m.model._engine.close()
    del m
    assert live() == before
