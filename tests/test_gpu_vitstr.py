"""GPU: ViTSTR (SURVEY.md 8f rank 3) through the strhub-compatible module -> C ABI -> the same sm_90a encoder kernels,
against the golden outputs of the reference's own strhub.models.vitstr.model.ViTSTR and the CPU oracle.
Tolerances: the bf16-operand contract of tests/test_gpu_parity.py (TOL_FP32_MAX / TOL_FP32_MEAN / TAU)."""
import glob
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = sorted(glob.glob(os.path.join(GOLDEN, "vitstr_*.pt")))
TOL_FP32_MAX = 2.0e-2
TOL_FP32_MEAN = 3.0e-3
TAU = 2.0e-2


def _model(seed, **over):
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config("vitstr", **over)
    sd = init_state_dict(cfg, seed)
    m = create_model("vitstr", **over)
    m.model.load_state_dict(sd)
    return cfg, sd, m.eval().to("cuda")


def _clear_decisions_identical(engine_logits, ref_logits, tau):
    top2 = ref_logits.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > tau
    same = engine_logits.argmax(-1) == ref_logits.argmax(-1)
    return bool(same[clear].all()), int(clear.sum())


@pytest.mark.parametrize("fuse", [None, 7], ids=["default", "fused_ln"])
@pytest.mark.parametrize("path", CASES, ids=lambda p: os.path.basename(p)[:-3])
def test_vs_reference_golden(path, fuse):
    from parseq_b200.weights import synth_images, state_dict_digest
    blob = torch.load(path, weights_only=False)
    cfg, sd, m = _model(blob["weight_seed"], **blob["overrides"])
    if fuse is not None:          # small batches take the unfused pair by default: force the fused GEMM+LN kernels too
        m.model.set_engine_option("fuse_ln", fuse)
    assert state_dict_digest(sd) == blob["sd_digest"]
    x = synth_images(cfg, blob["batch"], blob["image_seed"]).cuda()
    with torch.inference_mode():
        logits = m(x, blob["max_length"]).cpu()
        feats = m.model.forward_features(x[:1]).cpu()[0]
    ref = blob["logits"]
    assert logits.shape == ref.shape
    err = (logits - ref).abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN, (err.max().item(), err.mean().item())
    ok, n_clear = _clear_decisions_identical(logits, ref, TAU)
    assert ok, f"a clear (margin > {TAU}) decision differs ({n_clear} clear decisions)"
    ferr = (feats - blob["features0"]).abs()
    assert feats.shape == blob["features0"].shape            # [T + 1, D]: class token kept by forward_features
    assert ferr.max().item() <= 5e-2 and ferr.mean().item() <= 5e-3, (ferr.max().item(), ferr.mean().item())


def test_decisions_vs_live_fp32_oracle_and_batch_properties():
    from oracle.vitstr_oracle import VitstrOracle
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(22)
    x = synth_images(cfg, 70, 41)
    ref = VitstrOracle(cfg, sd, "fp32").system_forward(x[:24])
    xc = x.cuda()
    with torch.inference_mode():
        l1, i1 = m.model.forward_tokens(xc, None, return_ids=True)
        l2 = m(xc)
        l3 = m(xc[:5])
        l4 = m(xc, 9)
    assert l1.shape == (70, 26, 95) and torch.isfinite(l1).all()
    err = (l1[:24].cpu() - ref).abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN, (err.max().item(), err.mean().item())
    ok, n_clear = _clear_decisions_identical(l1[:24].cpu(), ref, TAU)
    assert ok and n_clear > 100
    assert torch.equal(l1, l2)                                # deterministic
    assert torch.equal(l1[:5], l3)                            # batch-composition invariance
    assert torch.equal(l1[:, :10], l4)                        # max_length only slices tokens (vitstr/system.py:66-70)
    assert torch.equal(i1.long(), l1.argmax(-1))


def test_uint8_input_and_postprocess():
    cfg, sd, m = _model(23)
    g = torch.Generator().manual_seed(5)
    u8 = torch.randint(0, 256, (6, 32, 128, 3), dtype=torch.uint8, generator=g)
    xf = (u8.permute(0, 3, 1, 2).to(torch.float32).div(255) - 0.5) / 0.5
    with torch.inference_mode():
        lf = m(xf.cuda())
        lu = m(u8.cuda())
        labels, confs = m.postprocess(lf)
        ref_labels, ref_probs = m.tokenizer.decode(lf.softmax(-1))
        res = m.test_step((xf.cuda(), ["a"] * 6), -1)["output"]
    assert torch.equal(lf, lu)
    assert labels == ref_labels
    assert max(abs(a - p.prod().item()) for a, p in zip(confs, ref_probs)) < 1e-6
    assert res.num_samples == 6


def test_too_few_patches_is_rejected_loudly():
    from parseq_b200.factory import create_model
    from parseq_b200.engine import EngineError
    m = create_model("vitstr", img_size=[32, 64], patch_size=[8, 8]).eval().to("cuda")     # 32 patches < 26 + 1? no: 32 >= 26
    with torch.inference_mode():
        assert m(torch.zeros(1, 3, 32, 64, device="cuda")).shape == (1, 26, 95)
    m = create_model("vitstr", img_size=[32, 32], patch_size=[8, 8]).eval().to("cuda")     # 16 patches < 26 kept tokens
    with pytest.raises(EngineError, match="at least max_label_length"):
        m(torch.zeros(1, 3, 32, 32, device="cuda"))
