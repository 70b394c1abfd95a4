"""Image geometries that put the PARSeq decoder in each image-token-count regime (shared by test_gpu_token_counts.py and
test_token_counts_cpu.py).  T = (H / ph) * (W / pw) image tokens, Kp = 3 * ph * pw is the K of the patch GEMM."""
from parseq_b200.config import make_config

# T -> (img_size, patch_size, Kp, what the geometry reaches first)
GEOMETRIES = {
    32: ((16, 64), (4, 8), 96, "cluster AR kernel with 64-row K/V boxes"),
    49: ((28, 28), (4, 4), 48, "64-row boxes, ragged; patch GEMM with K < 64"),
    64: ((32, 128), (4, 16), 192, "exactly one 64-row box"),
    65: ((20, 52), (4, 4), 48, "128-row box with 63 masked rows"),
    100: ((40, 80), (4, 8), 96, "ragged single 128-key block"),
    130: ((40, 104), (4, 8), 96, "second key block with 2 live keys"),
    256: ((32, 256), (4, 8), 96, "largest accepted T"),
}


def geometry_config(T, experiment="parseq", enc_depth=2):
    """(config, create_model overrides) of `experiment` at the geometry of T, with a shallow encoder."""
    img, patch, _, _ = GEOMETRIES[T]
    over = dict(img_size=img, patch_size=patch, enc_depth=enc_depth)
    return make_config(experiment, **over), over
