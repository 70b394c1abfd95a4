"""Tiny end-to-end run for compute-sanitizer (not a test):

    compute-sanitizer --tool memcheck|racecheck|synccheck python tests/sanitize_small.py

PARSeq-Ti and -S in every decode mode, with the kernels whose synchronisation crosses CTAs or proxies forced on: GEMM CTA
pairs (W tile multicast, remote empty-barrier arrivals), the fused residual-GEMM + LayerNorm in all three modes (single
CTA, multicast pair, column-split pair exchanging row statistics through distributed shared memory), the one-kernel MLP
on CTA pairs, the wgmma attention, the cluster AR kernel in both cluster sizes and the grid-barrier AR kernel, and
PARSeq.decode with masks."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.config import make_config
from parseq_b200.factory import create_model
from parseq_b200.weights import init_state_dict, synth_images

# (decode_ar, refine_iters, max_length, ar_kernel, ar_cluster_size, batch, launch options)
RUNS = [
    (True, 1, None, 2, 0, 3, {"fuse_ln": 7, "cta_group": 2, "attn_impl": 1}),
    (True, 0, 4, 2, 6, 19, {"fuse_ln": 7, "ln_cta_group": 2, "ln_split": 1}),
    (False, 2, None, 2, 0, 3, {"fuse_ln": 7, "fuse_mlp": 1, "mlp_cta_group": 2}),
    (True, 0, 4, 1, 0, 3, {"fuse_ln": 0}),
]

for exp in ("parseq-tiny", "parseq"):
    cfg = make_config(exp)
    sd = init_state_dict(cfg, 0)
    for ar, ri, ml, impl, cs, B, opts in RUNS:
        m = create_model(exp, decode_ar=ar, refine_iters=ri)
        m.model.load_state_dict(sd)
        m.model.set_engine_option("use_graph", 0)
        m.model.set_engine_option("ar_kernel", impl)
        m.model.set_engine_option("ar_cluster_size", cs)
        for k, v in opts.items():
            m.model.set_engine_option(k, v)
        m = m.eval().to("cuda")
        x = synth_images(cfg, B, 1).cuda()
        with torch.inference_mode():
            out = m(x, ml)
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        print("ok:", exp, "ar", ar, "refine", ri, "max_length", ml, "ar_kernel", impl, "cluster", cs, opts, tuple(out.shape), flush=True)
    # decode API with masks
    m = create_model(exp); m.model.load_state_dict(sd); m = m.eval().to("cuda")
    x = synth_images(cfg, 2, 3).cuda()
    with torch.inference_mode():
        mem = m.model.encode(x)
        tgt = torch.randint(1, 90, (2, 9), device="cuda"); tgt[:, 0] = 95
        qm = torch.triu(torch.ones((9, 9), dtype=torch.bool, device="cuda"), 1)
        out = m.model.head(m.model.decode(tgt, mem, tgt_query_mask=qm))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    print("ok:", exp, "decode + head", tuple(out.shape), flush=True)
print("sanitize_small done")
