"""CPU: every geometry of test_gpu_token_counts.py builds a config with the stated image-token count T and patch-GEMM
depth Kp, and the fp32 oracle runs a full AR + refine decode on it."""
import pytest
import torch

from token_count_geometries import GEOMETRIES, geometry_config


@pytest.mark.parametrize("experiment", ["parseq", "parseq-tiny", "parseq-base-48x160"])
@pytest.mark.parametrize("T", sorted(GEOMETRIES))
def test_geometry_has_stated_token_count_and_runs_in_oracle(T, experiment):
    from oracle.parseq_oracle import ParseqOracle
    from parseq_b200.weights import init_state_dict, synth_images
    _, _, Kp, _ = GEOMETRIES[T]
    cfg, _ = geometry_config(T, experiment, enc_depth=1)
    assert cfg.num_patches == T and cfg.enc_tokens == T and cfg.patch_dim == Kp
    assert 1 <= T <= 256 and Kp % 8 == 0           # the engine's limits (parseq_create)
    sd = init_state_dict(cfg, 0, sharp=4.0)
    assert tuple(sd["encoder.pos_embed"].shape) == (1, T, cfg.embed_dim)
    assert tuple(sd["encoder.patch_embed.proj.weight"].shape) == (cfg.embed_dim, 3, *cfg.patch_size)
    o = ParseqOracle(cfg, sd, "fp32").forward(synth_images(cfg, 2, T), 25, True, 1)
    assert o.memory.shape == (2, T, cfg.embed_dim)
    assert o.logits.shape == (2, 26, cfg.num_classes) and bool(torch.isfinite(o.logits).all())
