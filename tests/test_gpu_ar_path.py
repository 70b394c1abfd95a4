"""GPU: which implementation runs the AR loop - the cluster kernel (dec_ar2.cuh), the grid-barrier kernel (dec_ar.cuh) or
the chain of separate kernels - for head widths, label lengths, decoder shapes and the "ar_kernel" option.  One small eager
forward per case with device timing on: the cluster kernel records its cluster size, both persistent kernels time their
launch under the "dec_ar" category, and the chain launches nothing there."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# case: (head classes C, max_label_length (L - 1), dec_depth, dec_mlp_ratio, ar_kernel option or None, expected path)
CASES = {
    "c95":              (95,  25, 1, 4, None, "cluster"),
    "c96":              (96,  25, 1, 4, None, "cluster"),
    "c97":              (97,  25, 1, 4, None, "grid"),
    "c110_l26":         (110, 25, 1, 4, None, "grid"),
    "c110_l32":         (110, 31, 1, 4, None, "grid"),
    "c110_l33":         (110, 32, 1, 4, None, "chain"),
    "c110_l40":         (110, 39, 1, 4, None, "chain"),
    "c128":             (128, 25, 1, 4, None, "grid"),
    "c129":             (129, 25, 1, 4, None, "cluster"),
    "c200":             (200, 25, 1, 4, None, "cluster"),
    "c95_l64":          (95,  63, 1, 4, None, "cluster"),
    "c95_mlp8":         (95,  25, 1, 8, None, "grid"),
    "c200_mlp8":        (200, 25, 1, 8, None, "chain"),
    "c95_depth2":       (95,  25, 2, 4, None, "chain"),
    "c95_ar_kernel0":   (95,  25, 1, 4, 0,    "chain"),
    "c95_ar_kernel1":   (95,  25, 1, 4, 1,    "grid"),
    "c110_ar_kernel2":  (110, 25, 1, 4, 2,    "grid"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_ar_loop_implementation(case):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict, synth_images
    C, mll, depth, mlp, ar_kernel, want = CASES[case]
    kw = dict(dec_depth=depth, dec_mlp_ratio=mlp)
    cfg = make_config_long("parseq-tiny", mll, C - 95, **kw)
    m = create_model("parseq-tiny", charset_train=charset(C - 95), max_label_length=mll, decode_ar=True, refine_iters=1, **kw)
    m.model.load_state_dict(init_state_dict(cfg, 5))
    m = m.eval().to("cuda")
    assert cfg.num_classes == C
    eng = m.model.engine()
    if ar_kernel is not None:
        eng.set_option("ar_kernel", ar_kernel)
    eng.set_option("timing", 1)
    with torch.inference_mode():
        logits = m.model.forward(m.tokenizer, synth_images(cfg, 3, 6).cuda())
    torch.cuda.synchronize()
    ar_launches = eng.get_timing()["dec_ar"]["launches"]
    eng.set_option("timing", 0)
    assert logits.shape[0] == 3 and logits.shape[2] == C
    cluster_size = eng.debug_int("ar_last_cluster_size")
    got = "cluster" if cluster_size > 0 else ("grid" if ar_launches == 1 else "chain")
    assert got == want, (got, cluster_size, ar_launches)
    assert ar_launches == (0 if want == "chain" else 1)
