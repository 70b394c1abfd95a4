"""Raw crops of any size on the GPU (parseq_resize_crops, parseq_forward_crops, parseq_forward_host_crops):
  * the device resize is byte-identical to the reference transform's goldens and to live PIL (T.Resize(img_size,
    BICUBIC) after Image.rotate(r, expand=True)), at 32 x 128, 224 x 224 (ViTSTR) and 48 x 160;
  * model(crops) returns logits, ids and steps bitwise equal to model(golden floats) and to the uint8 path on the
    PIL-resized stack, for PARSeq-S and ViTSTR, AR + refine and refine_iters = 0 (early-exit length S), graph and eager,
    one crop, a few, two-half uploads (300) and more than max_batch;
  * the host variant equals the device variant; invalid metadata launches nothing."""
import numpy as np
import pytest
import torch

import crop_goldens

pytestmark = pytest.mark.gpu


def _model(experiment, seed=0, refine_iters=1, **kw):
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config(experiment, **kw)
    m = create_model(experiment, **({"refine_iters": refine_iters} if experiment != "vitstr" else {}), **kw)
    m.model.load_state_dict(init_state_dict(cfg, seed))
    return m.eval().to("cuda")


def _pil(img, size, rotation):
    from PIL import Image
    import torchvision.transforms as T
    pil = Image.fromarray(img)
    if rotation:
        pil = pil.rotate(rotation, expand=True)
    return np.asarray(T.Resize(size, T.InterpolationMode.BICUBIC)(pil))


def _ragged(n, seed):
    """Crop sizes of the benchmark's distribution: h in [16, 128], w in [32, 512]."""
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.integers(0, 256, (int(rng.integers(16, 129)), int(rng.integers(32, 513)), 3),
                                         dtype=np.uint8)) for _ in range(n)]


@pytest.fixture(scope="module")
def parseq():
    return _model("parseq")


@pytest.fixture(scope="module")
def vitstr():
    """ViTSTR at 224 x 224 (16 x 16 patches), the reference's ViTSTR image size."""
    return _model("vitstr", img_size=(224, 224), patch_size=(16, 16))


@pytest.mark.parametrize("name", crop_goldens.NAMES)
def test_resize_equals_goldens(parseq, vitstr, name):
    from oracle.make_golden_crops import digest
    crops, g = crop_goldens.load(name)
    dev = [torch.from_numpy(a).cuda() for a in crops]
    for (size, rotation), case in g["cases"].items():
        m = parseq if tuple(size) == (32, 128) else vitstr
        out = m.preprocess(dev, rotation).cpu().numpy()
        assert [digest(x) for x in out] == case["u8_sha256"], (name, size, rotation)


@pytest.mark.parametrize("rotation", [0, 90, 180, 270])
def test_resize_equals_live_pil(parseq, vitstr, rotation):
    """The CPU sweep's shapes (1-pixel sides, the tall-crop pass order, unchanged axes), 8192-pixel sides and a crop of
    the largest demo image's size, in one ragged batch, at 32 x 128, 224 x 224 and 48 x 160."""
    rng = np.random.default_rng(rotation)
    sizes = [(1, 1), (1, 300), (300, 1), (101, 1), (100, 1), (268, 2), (3000, 3), (32, 128), (90, 128), (224, 224),
             (224, 31), (64, 500), (17, 4000), (1, 8192), (8192, 1), (871, 1774), (48, 160)]
    sizes += [(int(rng.integers(1, 200)), int(rng.integers(1, 600))) for _ in range(16)]
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    crops = [torch.from_numpy(a).cuda() for a in imgs]
    m48 = _model("parseq", img_size=(48, 160))
    for m, size in ((parseq, (32, 128)), (vitstr, (224, 224)), (m48, (48, 160))):
        out = m.preprocess(crops, rotation).cpu().numpy()
        for i, a in enumerate(imgs):
            assert np.array_equal(out[i], _pil(a, size, rotation)), (size, sizes[i])


def _check_forward(m, crops, ref_u8, ref_float=None):
    """model(crops) == model(uint8 stack) (== model(float images) if given), logits and ids; steps through the shape."""
    inner = m.model
    with torch.inference_mode():
        if hasattr(inner, "refine_iters"):
            lc, ic = inner.forward(m.tokenizer, crops, None, return_ids=True)
            lu, iu = inner.forward(m.tokenizer, ref_u8.cuda(), None, return_ids=True)
        else:
            lc, ic = inner.forward_tokens(crops, None, return_ids=True)
            lu, iu = inner.forward_tokens(ref_u8.cuda(), None, return_ids=True)
        lf = m(ref_float.cuda()) if ref_float is not None else None
    assert lc.shape == lu.shape
    assert torch.equal(lc.cpu(), lu.cpu()) and torch.equal(ic.cpu(), iu.cpu())
    if lf is not None:
        assert torch.equal(lc.cpu(), lf.cpu())
    return lc, ic


@pytest.mark.parametrize("arch", ["parseq", "vitstr"])
@pytest.mark.parametrize("refine", [1, 0])
@pytest.mark.parametrize("graph", [1, 0], ids=["graph", "eager"])
def test_forward_crops_equals_golden_floats(arch, refine, graph):
    if arch == "vitstr" and refine == 0:
        pytest.skip("ViTSTR has no decoder")
    m = _model(arch, refine_iters=refine) if arch == "parseq" else _model(arch, img_size=(224, 224), patch_size=(16, 16))
    m.model.set_engine_option("use_graph", graph)
    crops, g = crop_goldens.load("demo" if arch == "parseq" else "seeded")
    size = (32, 128) if arch == "parseq" else (224, 224)
    ref_u8, ref_float = crop_goldens.reference_stack(crops, g, size, 0)
    _check_forward(m, [torch.from_numpy(a).cuda() for a in crops], ref_u8, ref_float)


@pytest.mark.parametrize("B", [1, 7, 300, 700])
@pytest.mark.parametrize("graph", [1, 0], ids=["graph", "eager"])
def test_forward_crops_batches(parseq, B, graph):
    """700 > max_batch (512): two super-chunks; 300 and the 512 chunk take the two-half upload on the host variant."""
    parseq.model.set_engine_option("use_graph", graph)
    try:
        rotation = 90 if B == 7 else 0
        crops = _ragged(B, B)
        ref = torch.stack([torch.from_numpy(_pil(c.numpy(), (32, 128), rotation)) for c in crops])
        with torch.inference_mode():
            lc, ic = parseq.model.forward(parseq.tokenizer, [c.cuda() for c in crops], None, return_ids=True,
                                          rotation=rotation)
            lu, iu = parseq.model.forward(parseq.tokenizer, ref.cuda(), None, return_ids=True)
            lh, ih = parseq.model.forward(parseq.tokenizer, crops, None, return_ids=True, rotation=rotation)
        assert torch.equal(lc.cpu(), lu.cpu()) and torch.equal(ic.cpu(), iu.cpu())
        assert lh.device.type == "cpu" and torch.equal(lh, lc.cpu()) and torch.equal(ih, ic.cpu())
    finally:
        parseq.model.set_engine_option("use_graph", 1)


def test_forward_crops_refine_zero_early_exit_and_vitstr_host():
    """refine_iters = 0 returns the S steps the batch ran, for crops as for the uint8 stack; ViTSTR host == device."""
    m = _model("parseq", refine_iters=0)
    crops = _ragged(40, 3)
    ref = torch.stack([torch.from_numpy(_pil(c.numpy(), (32, 128), 0)) for c in crops])
    lc, _ = _check_forward(m, [c.cuda() for c in crops], ref)
    with torch.inference_mode():
        lh = m(crops)
    assert torch.equal(lh, lc.cpu())
    v = _model("vitstr")
    vr = torch.stack([torch.from_numpy(_pil(c.numpy(), (32, 128), 0)) for c in crops])
    lvc, _ = _check_forward(v, [c.cuda() for c in crops], vr)
    with torch.inference_mode():
        assert torch.equal(v(crops), lvc.cpu())


def test_pil_images_take_the_host_variant(parseq):
    from PIL import Image
    crops = _ragged(5, 11)
    with torch.inference_mode():
        lp = parseq([Image.fromarray(c.numpy()) for c in crops])
        lc = parseq([c.cuda() for c in crops])
    assert lp.device.type == "cpu" and torch.equal(lp, lc.cpu())


def test_invalid_metadata_launches_nothing(parseq):
    from parseq_b200.engine import CropsC, EngineError
    eng = parseq.model.engine()
    data = torch.zeros(3 * 16 * 16, dtype=torch.uint8, device="cuda")
    offsets = torch.tensor([0, 0], dtype=torch.int64)
    out = torch.empty((2, 32, 128, 3), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    before = eng.launches
    for sizes, rot, nbytes in (([[16, 16], [16, 17]], 0, data.numel()),     # second crop past data_bytes
                               ([[16, 16], [0, 4]], 0, data.numel()),       # empty side
                               ([[16, 16], [16, 16]], 30, data.numel())):   # rotation
        sz = torch.tensor(sizes, dtype=torch.int32)
        c = CropsC(data.data_ptr(), nbytes, offsets.data_ptr(), sz.data_ptr(), rot)
        with pytest.raises(EngineError, match="error -1"):
            eng.resize_crops(c, 2, out.data_ptr(), st)
        logits = torch.empty((2, 26, 95), device="cuda")
        with pytest.raises(EngineError, match="error -1"):
            eng.forward_crops(c, 2, logits.data_ptr(), None, None, st)
    assert eng.launches == before
    with pytest.raises(ValueError):
        parseq([torch.zeros((4, 4, 3), dtype=torch.uint8), torch.zeros((4, 4, 3), dtype=torch.uint8, device="cuda")])
    with pytest.raises(RuntimeError):
        parseq([torch.zeros((0, 4, 3), dtype=torch.uint8, device="cuda")])
