"""Text regions of full frames on the GPU (parseq_warp_regions, crop_regions):
  * the device warp matches every golden digest of PIL's Image.transform(PERSPECTIVE, BICUBIC), also in a call of more
    regions than max_batch, and the coefficients it is given are the golden doubles;
  * integer boxes equal torch slicing of the frame (0 outside it); CPU and PIL frames give the bytes of CUDA frames;
  * every raw-crop path returns on the regions exactly what it returns on the same crops as separate CUDA tensors:
    forward (logits, ids and the step count, PARSeq-S, PARSeq-Ti without refinement, ViTSTR-S), per-crop rotations,
    read_oriented, score, beam_search(lexicon=) and locate;
  * to_frame sends each crop's corners back onto its quad."""
import math

import numpy as np
import pytest
import torch

import make_golden_regions as mg

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
def parseq_ti():
    return _model("parseq-tiny", refine_iters=0)


@pytest.fixture(scope="module")
def vitstr():
    return _model("vitstr", img_size=(224, 224), patch_size=(16, 16))


@pytest.fixture(scope="module")
def golden():
    return mg.load()


def _check_golden(rc, g):
    assert torch.equal(rc.coeffs.view(torch.int64), g["coeffs"].view(torch.int64))
    assert [tuple(c.shape[:2]) for c in rc] == [tuple(s) for s in g["sizes"]]
    got = [mg.digest(c.cpu().numpy()) for c in rc]
    bad = [i for i, (a, b) in enumerate(zip(got, g["sha256"])) if a != b]
    assert not bad, f"regions {bad} differ from PIL"


def test_warp_equals_goldens(parseq, golden):
    frames, g = golden
    with torch.inference_mode():
        rc = parseq.crop_regions([torch.from_numpy(f).cuda() for f in frames], g["quads"], frame_index=g["frame_index"])
    _check_golden(rc, g)


def test_warp_equals_goldens_past_max_batch(golden):
    frames, g = golden
    m = _model("parseq-tiny")
    m.model.set_engine_option("max_batch", 16)          # 53 regions: four chunks, the last one partial
    with torch.inference_mode():
        rc = m.crop_regions([torch.from_numpy(f).cuda() for f in frames], g["quads"], frame_index=g["frame_index"])
    _check_golden(rc, g)


def test_boxes_equal_slicing(parseq):
    frame = torch.from_numpy(mg.make_frame(200, 300, 11, 1)).cuda()
    boxes = [(0, 0, 300, 200), (37, 21, 137, 61), (299, 199, 300, 200), (-7, -3, 12, 9), (280, 190, 320, 230),
             (400, 10, 420, 30), (5, -50, 9, -40), (0, 0, 1, 1), (100, 20, 101, 180), (10, 150, 290, 151)]
    with torch.inference_mode():
        rc = parseq.crop_regions(frame, torch.tensor(boxes, dtype=torch.int64))
    pad = 64
    padded = torch.zeros((200 + 2 * pad, 300 + 2 * pad + 64, 3), dtype=torch.uint8, device="cuda")
    padded[pad:pad + 200, pad:pad + 300] = frame
    for (x0, y0, x1, y1), c in zip(boxes, rc):
        assert torch.equal(c, padded[y0 + pad:y1 + pad, x0 + pad:x1 + pad]), (x0, y0, x1, y1)
    assert torch.equal(rc.coeffs[:, [0, 1, 3, 4, 6, 7]],
                       torch.tensor([[1.0, 0.0, 0.0, 1.0, 0.0, 0.0]], dtype=torch.float64).expand(len(boxes), 6))


def test_cpu_and_pil_frames_equal_cuda_frames(parseq, golden):
    from PIL import Image
    frames, g = golden
    keep = [i for i, f in enumerate(g["frame_index"]) if f != 3]       # the 4K frame is covered on the device path
    fr = frames[:3] + frames[4:]
    index = [{0: 0, 1: 1, 2: 2, 4: 3}[g["frame_index"][i]] for i in keep]
    quads = g["quads"][keep]
    with torch.inference_mode():
        ref = parseq.crop_regions([torch.from_numpy(f).cuda() for f in fr], quads, frame_index=index)
        cpu = parseq.crop_regions([torch.from_numpy(f) for f in fr], quads, frame_index=index)
        pil = parseq.crop_regions([Image.fromarray(f) for f in fr], quads.numpy(), frame_index=np.array(index))
        one = parseq.crop_regions(torch.from_numpy(fr[1]), quads[[k for k, f in enumerate(index) if f == 1]])
    for a, b, c in zip(ref, cpu, pil):
        assert a.is_cuda and b.is_cuda and c.is_cuda
        assert torch.equal(a, b) and torch.equal(a, c)
    assert all(torch.equal(a, b) for a, b in zip([c for c, f in zip(ref, index) if f == 1], one))


def _workload(n, seed, shape=(480, 640)):
    """Seeded text-like regions (rotated by up to 45 degrees, mild perspective) of two blocky frames."""
    rng = np.random.default_rng(seed)
    H, W = shape
    frames = [torch.from_numpy(mg.make_frame(H, W, seed + k, 4)).cuda() for k in range(2)]
    quads, index = [], []
    while len(quads) < n:
        th = rng.uniform(-math.pi / 4, math.pi / 4)
        w, h = rng.uniform(40, 400), rng.uniform(16, 80)
        q = mg.rect(rng.uniform(0, W), rng.uniform(0, H), w, h, math.cos(th), math.sin(th))
        q = [(x + rng.uniform(-0.05, 0.05) * h, y + rng.uniform(-0.05, 0.05) * h) for x, y in q]
        if mg.convex(q):
            quads.append(q)
            index.append(len(quads) % 2)
    return frames, torch.tensor(quads, dtype=torch.float64), index


@pytest.fixture(scope="module")
def regions(parseq):
    frames, quads, index = _workload(40, 5)
    with torch.inference_mode():
        rc = parseq.crop_regions(frames, quads, frame_index=index)
    return rc, [c.clone() for c in rc]


def _eq(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_eq(x, y) for x, y in zip(a, b))
    return a == b


@pytest.mark.parametrize("name", ["parseq", "parseq_ti", "vitstr"])
def test_forward_on_regions_equals_separate_crops(request, regions, name):
    m = request.getfixturevalue(name)
    rc, sep = regions
    with torch.inference_mode():
        if name == "vitstr":
            a = m.model.forward_tokens(rc, return_ids=True)
            b = m.model.forward_tokens(sep, return_ids=True)
        else:
            a = m.model.forward(m.tokenizer, rc, return_ids=True)     # refine_iters 0: the length is the step count
            b = m.model.forward(m.tokenizer, sep, return_ids=True)
        rot = [(0, 90, 180, 270)[i % 4] for i in range(len(rc))]
        c, d = m(rc, rotation=rot), m(sep, rotation=rot)
    assert _eq(a, b) and a[0].is_cuda
    assert _eq(c, d)


def test_read_oriented_score_beam_and_locate_on_regions(parseq, vitstr, regions):
    rc, sep = regions
    words = ["text", "word", "hello", "a", "region"]
    with torch.inference_mode():
        for m in (parseq, vitstr):
            assert _eq(m.read_oriented(rc, min_confidence=0.5), m.read_oriented(sep, min_confidence=0.5))
            assert _eq(m.score(rc, words, return_token_logprobs=True), m.score(sep, words, return_token_logprobs=True))
            assert _eq(m.beam_search(rc, 3, lexicon=words), m.beam_search(sep, 3, lexicon=words))
        assert _eq(parseq.locate(rc), parseq.locate(sep))
        assert _eq(parseq.locate(rc, text="word"), parseq.locate(sep, text="word"))
        assert _eq(parseq.lexicon_decode(rc, words), parseq.lexicon_decode(sep, words))


def test_to_frame_returns_the_quads(regions):
    rc, _ = regions
    for i, c in enumerate(rc):
        h, w = c.shape[:2]
        corners = rc.to_frame(torch.tensor([[0.0, 0.0], [w, 0.0], [w, h], [0.0, h]]), i)
        scale = max(1.0, float(rc.quads[i].abs().max()))
        assert float((corners - rc.quads[i]).abs().max()) <= 1e-9 * scale, i


def test_locate_centres_map_into_the_frame(parseq, regions):
    """locate's centres are crop pixels: to_frame puts them inside their region's quad."""
    rc, _ = regions
    with torch.inference_mode():
        _, _, centers, _ = parseq.locate(rc)
    for i, c in enumerate(centers):
        if len(c) == 0:
            continue
        p = rc.to_frame(c.double().cpu(), i)
        q = rc.quads[i]
        for k in range(4):                    # the same side of every edge as the quad's interior
            a, b = q[k], q[(k + 1) % 4]
            cross = (b[0] - a[0]) * (p[:, 1] - a[1]) - (b[1] - a[1]) * (p[:, 0] - a[0])
            assert bool((cross >= -1e-6).all()), (i, k)
