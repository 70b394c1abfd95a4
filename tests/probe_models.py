"""Probe models: real PARSeq / ViTSTR geometries whose weights and images make one detail of the arithmetic decide the
output by O(1).  TEST HELPER.

The error budgets of tests/encoder_reference.py and tests/decoder_reference.py are statistical: on random weights a
correct engine's bf16 rounding flips reach most outputs, and at D >= 384 or depth 2 some small bugs (an extra or a
missing key, a wrong LayerNorm eps, the tanh GELU, a bf16-rounded cross query) move the outputs no more than those flips
do.  A probe removes the noise floor instead of averaging over it.  Its residual stream is a +-1 pattern (or a pattern
of amplitude delta with a row variance comparable to the LayerNorm eps), so every LayerNorm output is exact in bf16, and
every sub-layer but the site under test adds exactly zero.  The site writes its result by flipping the signs of one
channel pair (+1, -1) -> (-1, +1) of the residual stream, which leaves the row a +-1 pattern when the arithmetic is
right and leaves it off that pattern by O(1) when it is not; or, for the eps probes, by a gate whose score moves by
more than 100 between the two eps, so that the site adds exactly zero on one side and O(1) on the other.  A correct
engine then agrees with the fp64 rounding-point model to fp32 rounding of a few sums (~1e-6), and each bug it covers
moves the output by 7e-3 to 26.

The expected output is always the fp64 model of the probe's weights; nothing is derived by hand.  GEMM weights are
bf16-exact (save the one row of `vitstr_rounding` that tests the rounding at load), biases and LayerNorm parameters are
fp32, and no probe produces NaN or inf.

Channels come in pairs (2m, 2m + 1) holding (s, -s), so every row has mean 0 and variance amp^2 exactly.  Pair 0 marks
the key a probe makes win or lose (the last token, +1 there only), pair 1 the 15 tied keys of the attention probe,
pairs 2 + 4 l .. 5 + 4 l are the flip pairs of block / layer l (+1 on every token), the rest a seeded pattern shared
by all tokens.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F

from decoder_reference import DecoderReference, DepthDecoderReference, engine_gelu, forced_ar_ids, refine_context
from encoder_reference import EncoderReference

EXPERIMENT = {192: "parseq-tiny", 384: "parseq", 768: "parseq-base-48x160", "vitstr": "vitstr", "vitstr-tail": "vitstr"}
N_TIED = 15                     # bf16(1/15) * 15 - 1 = +0.34 %
L_TAIL = 26
_KEY, _TIED = 0, 1              # indicator pairs


def _flip_pair(l: int, i: int) -> int:
    return 2 + 4 * l + i


def _bf(x) -> torch.Tensor:
    return torch.as_tensor(x, dtype=torch.float64).to(torch.bfloat16).to(torch.float32)


def _pattern(N: int, D: int, seed: int, tied=()) -> torch.Tensor:
    """[N, D] rows of +-1 in (s, -s) pairs: pair 0 is +1 on token N - 1 only, pair 1 on the tokens `tied` only, the flip
    pairs +1 everywhere, the others a seeded pattern shared by all tokens."""
    g = torch.Generator().manual_seed(seed)
    half = (torch.randint(0, 2, (D // 2,), generator=g) * 2 - 1).float()
    half[_flip_pair(0, 0): _flip_pair(2, 0)] = 1.0
    s = half.repeat(N, 1)
    s[:, _KEY] = -1.0
    s[-1, _KEY] = 1.0
    s[:, _TIED] = -1.0
    s[list(tied), _TIED] = 1.0
    return torch.stack([s, -s], dim=-1).reshape(N, D)


def _shared(D: int, seed: int) -> torch.Tensor:
    """The shared pattern of _pattern with the indicator pairs zeroed: the direction a gate reads."""
    s = _pattern(1, D, seed)[0].clone()
    s[: 2 * (_TIED + 1)] = 0.0
    return s


def _flip(W, b, pair: int, cols, w, total: float):
    """Rows 2 pair and 2 pair + 1 of (W, b) add +-(sum(w * o[cols]) - total - 2), w a scalar or one weight per column:
    (+1, -1) becomes (-1, +1) when sum(w * o[cols]) is `total`, as it is for a correct engine."""
    r = 2 * pair
    W[r, cols] = w
    W[r + 1, cols] = -w
    b[r] = -total - 2.0
    b[r + 1] = total + 2.0


@dataclass
class Probe:
    name: str
    key: tuple                          # the budget key: (embed_dim, depth), ("vitstr", 2) or ("vitstr-tail", 2)
    cfg: object
    sd: dict
    images: torch.Tensor
    covers: List[Tuple[str, tuple]]     # (BUGS name, budget key)
    tol: float                          # max |engine - model| a correct engine stays within
    decoder: bool = False
    forced: Optional[torch.Tensor] = None
    context: Optional[torch.Tensor] = None
    over: dict = field(default_factory=dict)    # create_model overrides
    # BUGS name -> the decoder passes it moves (DEC_PASSES names); a bug not listed moves every pass, and the passes a
    # listed bug leaves out stay bit-identical in the fp64 model
    moves: dict = field(default_factory=dict)

    # -- the fp64 model and the output it is compared on ----------------------------------------------------------------
    def encoder_model(self, accum=torch.float64, bug=None, device="cpu"):
        return EncoderReference(self.cfg, self.sd, accum=accum, device=device,
                                bug=None if self.decoder else bug)

    def memory(self, device="cpu"):
        """The bf16 encoder memory the decoder reads (a +-1 pattern for every decoder probe)."""
        return self.encoder_model(device=device).encode(self.images).to(torch.bfloat16).to(torch.float32)

    def expected(self, accum=torch.float64, bug=None, device="cpu", pass_="ar", cluster=False, memory=None):
        if not self.decoder:
            m = self.encoder_model(accum, bug, device)
            return m.tail(self.images, L_TAIL) if self.key[0] == "vitstr-tail" else m.encode(self.images)
        mem = self.memory(device) if memory is None else memory
        cls = DepthDecoderReference if self.cfg.dec_depth > 1 else DecoderReference
        m = cls(self.cfg, self.sd, accum=accum, device=device, bug=bug, cluster=cluster)
        if pass_ == "ar":
            return m.ar(mem, self.forced)
        if pass_ == "refine":
            return m.refine(mem, self.context)
        return m.nar(mem, self.cfg.max_label_length + 1)

    def score_terms(self, logits=None, **kw):
        """The terms `score` returns for the teacher-forced candidates of the AR pass: candidate b is forced[b, 1:] up to
        its first EOS (c_1..c_n), and term i <= n is log_softmax(logits[b, i])[t_i] with t = (c_1..c_n, EOS); 0 past n."""
        lg = self.expected(pass_="ar", **kw) if logits is None else logits
        return teacher_forced_terms(lg, self.forced)


def teacher_forced_terms(logits: torch.Tensor, forced: torch.Tensor) -> torch.Tensor:
    """[B, L] terms of the AR logits [B, L, C] under teacher forcing `forced` [B, L] (BOS first): see Probe.score_terms."""
    B, L, _ = logits.shape
    f = forced.to(logits.device).long()
    t = torch.cat([f[:, 1:], torch.zeros_like(f[:, :1])], dim=1)          # EOS = 0 after the last position
    eos = (t == 0).int()
    n = torch.where(eos.any(1), eos.argmax(1), torch.full((B,), L - 1, device=f.device))
    t[torch.arange(B), n] = 0
    lp = torch.log_softmax(logits.double(), dim=-1).gather(-1, t[..., None])[..., 0]
    return torch.where(torch.arange(L, device=f.device)[None] <= n[:, None], lp, torch.zeros_like(lp))


# ---- the encoder --------------------------------------------------------------------------------------------------
def _enc_names(cfg):
    return (lambda k: k) if cfg.arch == "vitstr" else (lambda k: "encoder." + k)


def _encoder_base(cfg, seed: int, amp: float, tied=()):
    """init_state_dict with every encoder block adding exactly zero, the patch embedding zero (or set by the caller),
    the LayerNorms the identity and the residual stream amp * _pattern: (state dict, name map, pattern)."""
    from parseq_b200.weights import init_state_dict
    sd = {k: v.clone() for k, v in init_state_dict(cfg, seed).items()}
    n = _enc_names(cfg)
    vit = cfg.arch == "vitstr"
    N = cfg.num_patches + (1 if vit else 0)
    pat = _pattern(N, cfg.embed_dim, seed, tied)
    sd[n("patch_embed.proj.weight")].zero_()
    sd[n("patch_embed.proj.bias")].zero_()
    sd[n("pos_embed")] = (amp * pat)[None].float()
    if vit:
        sd["cls_token"].zero_()
    for i in range(cfg.enc_depth):
        for k in ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2"):
            sd[n(f"blocks.{i}.{k}.weight")].zero_()
            sd[n(f"blocks.{i}.{k}.bias")].zero_()
        for k in ("norm1", "norm2"):
            sd[n(f"blocks.{i}.{k}.weight")].fill_(1.0)
            sd[n(f"blocks.{i}.{k}.bias")].zero_()
    sd[n("norm.weight")].fill_(1.0)
    sd[n("norm.bias")].zero_()
    if vit:
        _loud_head(sd, cfg.enc_depth)
    return sd, n, pat


def _loud_head(sd, depth, classwise=False):
    """Head columns of the flip pairs at +-1/4, so that a flip moves every logit by 1.  classwise: the column of flip
    pair (l, i) is +1/4 for class c when bit (4 l + i) mod 6 of c is set and -1/4 otherwise, so that a flip moves the
    classes' logits apart and log_softmax (scoring) sees it; every logit still moves by 1."""
    W = sd["head.weight"]
    c = torch.arange(W.shape[0])
    for l in range(depth):
        for i in range(4):
            r = 2 * _flip_pair(l, i)
            w = torch.where((c >> ((4 * l + i) % 6)) & 1 == 1, 0.25, -0.25) if classwise else 0.25
            W[:, r] = w
            W[:, r + 1] = -w


def _config(key, **over):
    from parseq_b200.config import make_config
    return make_config(EXPERIMENT[key[0]], enc_depth=key[1], **over)


def _images(cfg, B=2, seed=0):
    from parseq_b200.weights import synth_images
    return synth_images(cfg, B, 900 + seed)


def _enc_covers(key, bugs):
    return [(b, key) for b in bugs]


def enc_attention(key, seed=1) -> Probe:
    """Every block l: head 0's query is its bias alone, the last token the best key at score -64 and every other one at
    -256, v = 1 on the best key and 0 elsewhere; head 1's 15 tied keys score -8 and the rest -136, v = 1.5 everywhere.
    Head 0 flips pair (l, 0); head 1 adds 48 to pair (l, 1) against a bias of -50.  An extra zero key (score 0) takes
    head 0's weight, a dropped last key leaves head 0 the mean of v = 0, and P normalised before rounding returns
    bf16(1.5 * 15 * bf16(1/15)) = 1.5078 from head 1: every output of pair (l, 1) moves by 0.25 / sigma."""
    cfg = _config(key)
    N = cfg.num_patches + (1 if cfg.arch == "vitstr" else 0)
    tied = [(7 * i + 3) % (N - 1) for i in range(N_TIED)]
    assert len(set(tied)) == N_TIED
    sd, n, _ = _encoder_base(cfg, seed, 1.0, tied)
    D, h = cfg.embed_dim, cfg.enc_num_heads
    d = D // h
    scale = d ** -0.5
    for l in range(cfg.enc_depth):
        W, b = sd[n(f"blocks.{l}.attn.qkv.weight")], sd[n(f"blocks.{l}.attn.qkv.bias")]
        b[0] = 1.0 / scale                                   # head 0: q = e_0
        W[D, 2 * _KEY], b[D] = 96.0, -160.0                  # k_0 = 96 s_key - 160: -64 / -256
        W[2 * D: 2 * D + d, 2 * _KEY], b[2 * D: 2 * D + d] = 0.5, 0.5      # v = 1 / 0
        b[d] = 1.0 / scale                                   # head 1
        W[D + d, 2 * _TIED], b[D + d] = 64.0, -72.0          # k_0 = -8 / -136
        b[2 * D + d: 2 * D + 2 * d] = 1.5
        Wp, bp = sd[n(f"blocks.{l}.attn.proj.weight")], sd[n(f"blocks.{l}.attn.proj.bias")]
        _flip(Wp, bp, _flip_pair(l, 0), slice(0, d), 2.0 / d, 2.0)
        _flip(Wp, bp, _flip_pair(l, 1), slice(d, 2 * d), 0.5, 0.5 * 1.5 * d)
    covers = _enc_covers(key, ("attn_extra_zero_key", "attn_drop_last_key", "attn_p_normalised_before_rounding"))
    return Probe(f"enc_attention-{_kname(key)}", key, cfg, sd, _images(cfg), covers, 1e-4)


def gelu_points() -> Tuple[torch.Tensor, torch.Tensor]:
    """bf16 points b in [-6, 6] where bf16 of the engine's GELU, in fp32 and in fp64, and of the exact erf-GELU agree,
    1e-5 (relative) or more from a bf16 rounding boundary, and bf16 of the tanh GELU does not: (b, sign of the tanh
    form's step)."""
    x = torch.arange(-6.0, 6.0, 2.0 ** -9, dtype=torch.float64).to(torch.bfloat16).unique().double()
    r = lambda t: t.to(torch.bfloat16).double()
    e64 = engine_gelu(x)
    e32 = engine_gelu(x.float()).double()
    erf, tanh = F.gelu(x), F.gelu(x, approximate="tanh")
    step = torch.exp2(torch.floor(torch.log2(r(e64).abs().clamp(min=2.0 ** -126))) - 7)
    room = step / 2 - (e64 - r(e64)).abs()                 # distance to the nearest rounding boundary
    ok = (r(e64) == r(e32)) & (r(e64) == r(erf)) & (r(tanh) != r(erf)) & (room > 1e-5 * e64.abs())
    return x[ok].float(), torch.sign(r(tanh) - r(erf))[ok].float()


def enc_gelu(key, seed=2) -> Probe:
    """Every block l: attention zero, fc1's weight zero and its bias at gelu_points (so the hidden value is
    bf16(GELU(b)) exactly), fc2 summing them, each with the sign of the tanh form's step, into flip pair (l, 0).  The
    tanh GELU moves every hidden value by one bf16 step in the same direction of the sum."""
    cfg = _config(key)
    sd, n, _ = _encoder_base(cfg, seed, 1.0)
    pts, sgn = gelu_points()
    H = cfg.embed_dim * cfg.enc_mlp_ratio
    idx = torch.arange(H) % pts.numel()
    b1, w = pts[idx], sgn[idx] * 2.0 ** -6
    hid = engine_gelu(b1.double()).to(torch.bfloat16).double()
    total = float((hid * w.double()).sum())
    for l in range(cfg.enc_depth):
        sd[n(f"blocks.{l}.mlp.fc1.bias")] = b1.clone()
        W2, b2 = sd[n(f"blocks.{l}.mlp.fc2.weight")], sd[n(f"blocks.{l}.mlp.fc2.bias")]
        _flip(W2, b2, _flip_pair(l, 0), slice(None), w, total)
    covers = _enc_covers(key, ("gelu_tanh",))
    return Probe(f"enc_gelu-{_kname(key)}", key, cfg, sd, _images(cfg), covers, 1e-4)


def _ln_amplitude(eps: float, eps_bug: float, gain: float = 0.8125):
    """(delta, gain, gain_bug): the fp32 amplitude delta whose LayerNorm gain delta / sqrt(delta^2 + eps) is the bf16
    value `gain`, and the gain under eps_bug."""
    dl = float(torch.tensor(math.sqrt(eps * gain * gain / (1 - gain * gain)), dtype=torch.float32))
    return dl, dl / math.sqrt(dl * dl + eps), dl / math.sqrt(dl * dl + eps_bug)


def enc_ln_eps(key, seed=3) -> Probe:
    """The residual stream at amplitude delta (row variance delta^2 ~ 2e-6), where eps 1e-5 instead of 1e-6 halves the
    LayerNorm gain (0.81 -> 0.40).  Every block l: head 0's query reads norm1's gain through the shared pattern and
    scores the last token's key 113 or more below the others when the gain is right (so head 0 adds exactly zero) and
    above them when it is not; fc1's row 0 reads norm2's gain the same way, a GELU that is ~0 or ~5.  The final norm's
    gain is the output itself."""
    cfg = _config(key)
    eps, eps_bug = 1e-6, 1e-5
    dl, A, Ab = _ln_amplitude(eps, eps_bug)
    sd, n, _ = _encoder_base(cfg, seed, dl)
    D, h = cfg.embed_dim, cfg.enc_num_heads
    d = D // h
    s = _shared(D, seed)
    Ah, Abh = float(_bf(A)), float(_bf(Ab))
    mid = (Ah + Abh) / 2
    ns = float(s.abs().sum())
    for l in range(cfg.enc_depth):
        W, b = sd[n(f"blocks.{l}.attn.qkv.weight")], sd[n(f"blocks.{l}.attn.qkv.bias")]
        # q_0 (scaled) = g (gain - mid) with g < 0; k_0 = kappa gain s_key: the last token's score is q_0 * 2 kappa gain
        # above the others', at least 120 below them at the right gain and 120 above them at the bug's
        kappa = 64.0
        g = -120.0 / (2 * kappa * Abh) / min(Ah - mid, mid - Abh)
        w = float(_bf(g * d ** 0.5 / ns))
        W[0] = w * s
        b[0] = -w * ns * mid
        W[D, 2 * _KEY] = kappa
        W[2 * D: 2 * D + d, 2 * _KEY] = 0.5
        b[2 * D: 2 * D + d] = 0.5 * Ah                       # v = 0 off the last token at the right gain
        Wp, bp = sd[n(f"blocks.{l}.attn.proj.weight")], sd[n(f"blocks.{l}.attn.proj.bias")]
        Wp[2 * _flip_pair(l, 0), :d] = 2.0 ** -4
        # fc1 row 0: g1 (gain - mid), <= -12 at the right gain and >= 12 at the bug's
        W1, b1 = sd[n(f"blocks.{l}.mlp.fc1.weight")], sd[n(f"blocks.{l}.mlp.fc1.bias")]
        g1 = float(_bf(-12.0 / min(Ah - mid, mid - Abh) / ns))
        W1[0] = g1 * s
        b1[0] = -g1 * ns * mid
        sd[n(f"blocks.{l}.mlp.fc2.weight")][2 * _flip_pair(l, 1), 0] = 0.25
    covers = _enc_covers(key, ("ln_eps",))
    return Probe(f"enc_ln_eps-{_kname(key)}", key, cfg, sd, _images(cfg), covers, 1e-4)


def vitstr_rounding(key, seed=4) -> Probe:
    """ViTSTR with every pixel 1/2 + 3/4 of a bf16 step (rounded to nearest: 1/2 + 2^-8, truncated: 1/2) and the patch
    embedding's flip-pair rows summing all 96 pixels of a patch: row pair 0 with weight 1/8, row pair 1 with
    1/8 (1 + 3/4 2^-7) (bf16 at load: 1/8 (1 + 2^-7), truncated: 1/8).  Truncated patches move pair 0 by 0.047 and
    truncated weights pair 1 by 0.047."""
    cfg = _config(key)
    sd, n, _ = _encoder_base(cfg, seed, 1.0)
    K = 3 * cfg.patch_size[0] * cfg.patch_size[1]
    px = 0.5 + 0.75 * 2.0 ** -8
    w1 = 0.125 * (1 + 0.75 * 2.0 ** -7)
    W = sd["patch_embed.proj.weight"].view(cfg.embed_dim, K)
    b = sd["patch_embed.proj.bias"]
    pxr = 0.5 + 2.0 ** -8
    _flip(W, b, _flip_pair(0, 0), slice(None), 0.125, K * pxr * 0.125)
    _flip(W, b, _flip_pair(0, 1), slice(None), w1, K * pxr * 0.125 * (1 + 2.0 ** -7))
    img = torch.full((2, 3, cfg.img_size[0], cfg.img_size[1]), px, dtype=torch.float32)
    covers = _enc_covers(key, ("patch_round_trunc", "weight_round_trunc"))
    return Probe(f"vitstr_rounding-{_kname(key)}", key, cfg, sd, img, covers, 1e-4)


# ---- the decoder --------------------------------------------------------------------------------------------------
# image-token counts of the cross-attention probe besides token_count_geometries': T = 240 (12 x 20 patches) puts the
# last key inside the cluster kernel's second 128-row K/V box with 16 rows past it
EXTRA_GEOMETRIES = {240: ((48, 160), (4, 8))}


def _decoder_base(key, seed, amp, T=None, extra_chars=0, mll=25):
    """A PARSeq model at `key` whose encoder memory is the +-1 pattern (bf16-exact; pair 0 marks the last image token)
    and whose decoder layers add exactly zero, with the query stream amp * the shared pattern (every position alike).
    T: the image-token count (the width's own geometry if None); extra_chars: classes beyond the 95 of the default
    charset; mll: max_label_length."""
    from make_golden_long import charset
    from parseq_b200.config import make_config
    from token_count_geometries import GEOMETRIES
    D, depth = key
    over = dict(enc_depth=1, dec_depth=depth)
    if T is not None:
        img, patch = EXTRA_GEOMETRIES[T] if T in EXTRA_GEOMETRIES else GEOMETRIES[T][:2]
        over.update(img_size=img, patch_size=patch)
    if extra_chars:
        over["charset_train"] = charset(extra_chars)
    if mll != 25:
        over["max_label_length"] = mll
    cfg = make_config(EXPERIMENT[D], **over)
    sd, _, _ = _encoder_base(cfg, seed, 1.0)
    for l in range(depth):
        p = f"decoder.layers.{l}."
        for k in ("self_attn.in_proj_", "self_attn.out_proj.", "cross_attn.in_proj_", "cross_attn.out_proj.",
                  "linear1.", "linear2."):
            sd[p + k + "weight"].zero_()
            sd[p + k + "bias"].zero_()
        for k in ("norm1", "norm2", "norm_q", "norm_c"):
            sd[p + k + ".weight"].fill_(1.0)
            sd[p + k + ".bias"].zero_()
    sd["decoder.norm.weight"].fill_(1.0)
    sd["decoder.norm.bias"].zero_()
    L = cfg.max_label_length + 1
    s = _pattern(1, D, seed)[0]
    s[: 2 * (_TIED + 1)] = torch.tensor([1.0, -1.0, 1.0, -1.0])
    sd["pos_queries"] = (amp * s).expand(1, L, D).clone()
    _loud_head(sd, depth, classwise=True)
    return cfg, sd, over


def _dec_probe(name, key, cfg, sd, covers, tol, over, seed, B=2, ctx=None, moves=None) -> Probe:
    L, C = cfg.max_label_length + 1, cfg.num_classes
    bos = cfg.num_tokens - 2
    forced = forced_ar_ids(B, L, C, bos, 100 + seed)
    if ctx is None:
        ctx = refine_context(B, L, C, bos, [3, None], 200 + seed)
    tag = (f"-T{cfg.num_patches}" if "img_size" in over else "") + (f"-C{C}" if "charset_train" in over else "") + \
        (f"-L{L}" if "max_label_length" in over else "")
    return Probe(f"{name}-{_kname(key)}{tag}", key, cfg, sd, _images(cfg, B), covers, tol, decoder=True, forced=forced,
                 context=ctx, over=over, moves=moves or {})


def dec_cross(key, T=None, extra_chars=0, mll=25, seed=5) -> Probe:
    """Every layer l, cross-attention with queries from the bias alone.  Head 0: the last image token's key scores -64,
    every other -256, v = 1 on it and 0 elsewhere: flips pair (l, 0).  An extra zero key (score 0) takes the weight, a
    dropped last key leaves the mean of v = 0.  Head 1: q = (1 + 2^-9, -1, 1) against keys 2^13 (s, s) and -8 s of the
    indicator s: the last token scores 8 and the others -8, but 2^14 * 2^-9 = 32 of that gap sits in q's bits below bf16,
    so a bf16 q scores the last token -8 and the others +8: flips pair (l, 1) or not."""
    cfg, sd, over = _decoder_base(key, seed, 1.0, T, extra_chars, mll)
    D, h = cfg.embed_dim, cfg.dec_num_heads
    d = D // h
    rs = math.sqrt(d)
    for l in range(cfg.dec_depth):
        p = f"decoder.layers.{l}.cross_attn."
        W, b = sd[p + "in_proj_weight"], sd[p + "in_proj_bias"]
        c = 2 * _KEY
        b[0] = 1.0 * rs
        W[D, c], b[D] = 96.0, -160.0
        W[2 * D: 2 * D + d, c], b[2 * D: 2 * D + d] = 0.5, 0.5
        b[d], b[d + 1], b[d + 2] = (1 + 2.0 ** -9) * rs, -1.0 * rs, 1.0 * rs
        W[D + d, c], W[D + d + 1, c], W[D + d + 2, c] = 2.0 ** 13, 2.0 ** 13, -8.0
        W[2 * D + d: 2 * D + 2 * d, c], b[2 * D + d: 2 * D + 2 * d] = 0.5, 0.5
        Wo, bo = sd[p + "out_proj.weight"], sd[p + "out_proj.bias"]
        _flip(Wo, bo, _flip_pair(l, 0), slice(0, d), 2.0 / d, 2.0)
        _flip(Wo, bo, _flip_pair(l, 1), slice(d, 2 * d), 2.0 / d, 2.0)
    covers = [(bug, key) for bug in ("cross_extra_zero_key", "cross_drop_last_key", "cross_q_bf16")]
    return _dec_probe("dec_cross", key, cfg, sd, covers, 1e-4, over, seed)


def dec_ln_eps(key, T=None, extra_chars=0, mll=25, seed=6) -> Probe:
    """The query stream at amplitude delta (row variance ~ 2e-5), where eps 1e-6 instead of 1e-5 raises the LayerNorm
    gain from 0.81 to 0.98.  Every layer l: cross head 0's query reads norm1's gain through the shared pattern and scores
    the last image token 113 or more below the others at the right gain (v = 0 there: the head adds exactly zero) and
    above them at the bug's; linear1's row 0 reads norm2's gain, a GELU ~0 or ~5.  decoder.norm's gain reaches the head
    directly."""
    cfg, sd, over = _decoder_base(key, seed, 1.0, T, extra_chars, mll)
    eps, eps_bug = 1e-5, 1e-6
    dl, A, Ab = _ln_amplitude(eps, eps_bug)
    D, h = cfg.embed_dim, cfg.dec_num_heads
    d = D // h
    s = sd["pos_queries"][0, 0].clone()
    s[: 2 * (_TIED + 1)] = 0.0
    sd["pos_queries"] = (dl * sd["pos_queries"]).float()
    Ah, Abh = float(_bf(A)), float(_bf(Ab))
    mid = (Ah + Abh) / 2
    ns = float(s.abs().sum())
    kappa = 64.0
    for l in range(cfg.dec_depth):
        p = f"decoder.layers.{l}."
        W, b = sd[p + "cross_attn.in_proj_weight"], sd[p + "cross_attn.in_proj_bias"]
        # q_0 (scaled) = g (gain - mid); the last image token's score is q_0 * 2 kappa above the others', at least 120
        # below them at the right gain and 120 above them at the bug's
        g = 120.0 / (2 * kappa) / min(mid - Ah, Abh - mid)
        w = float(_bf(g * math.sqrt(d) / ns))
        W[0] = w * s
        b[0] = -w * ns * mid
        W[D, 2 * _KEY] = kappa
        W[2 * D: 2 * D + d, 2 * _KEY], b[2 * D: 2 * D + d] = 0.5, 0.5
        sd[p + "cross_attn.out_proj.weight"][2 * _flip_pair(l, 0), :d] = 2.0 ** -4
        g1 = float(_bf(12.0 / min(mid - Ah, Abh - mid) / ns))
        sd[p + "linear1.weight"][0] = g1 * s
        sd[p + "linear1.bias"][0] = -g1 * ns * mid
        sd[p + "linear2.weight"][2 * _flip_pair(l, 1), 0] = 0.25
    sd["head.weight"][:8] = 2.0 ** -4 * s
    return _dec_probe("dec_ln_eps", key, cfg, sd, [("ln_eps", key)], 1e-4, over, seed)


# ---- the decoder self-attention --------------------------------------------------------------------------------------
# pairs of the self-attention probes: a 7-bit position code (bit j on pair _CODE + j) and one token-indicator pair
_CODE, _NBITS = _flip_pair(2, 0), 7
_TOK = _CODE + _NBITS
SELF_B = 7                      # images per self-attention probe, each with its own ids and its own first EOS
SELF_EOS = {26: (3, 1, 12, 24, 25, 8, None), 64: (1, 31, 32, 33, 63, 8, None)}     # first EOS of image b (b mod 7)
_AR, _REFINE, _NAR = ("ar", "ar-cluster", "score"), ("refine",), ("nar",)


def marked(ids: torch.Tensor) -> torch.Tensor:
    """The token indicator of dec_self_order: odd ids (EOS = 0 is unmarked, BOS has its own row)."""
    return ids % 2 == 1


def self_context(B, L, C, bos, first_eos, seed):
    """Refinement contexts [B, L] without EOS but at first_eos[b % len(first_eos)] (None: no EOS).  Where the last key
    has the parity of the key before the first EOS, it is an EOS too, so that the latest key a padding mask with a hole
    lets through has the other parity."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, max(C, 2), (B, L), generator=g, dtype=torch.int32)
    for b in range(B):
        e = first_eos[b % len(first_eos)]
        if e is not None:
            ids[b, e] = 0
            if e < L - 2 and (L - 1) % 2 == (e - 1) % 2:
                ids[b, L - 1] = 0
    ids[:, 0] = bos
    return ids


def _self_rows(sd, cfg):
    """pos_queries[j] carries the code of j + 1 on the code pairs and -1 on the token pair; BOS's embedding the full row
    with code 0, every other token's embedding +-2 on the token pair where marked() and 0 elsewhere, so that context row
    k (BOS, or sqrt(D) E[id] + pos_queries[k - 1]) is a +-1 pattern whose code is k and whose token pair is +1 on
    marked ids."""
    D = cfg.embed_dim
    L = cfg.max_label_length + 1
    s = sd["pos_queries"][0].view(L, D // 2, 2)[:, :, 0].clone()       # every row the shared pattern
    for j in range(_NBITS):
        s[:, _CODE + j] = torch.tensor([1.0 if ((q + 1) >> j) & 1 else -1.0 for q in range(L)])
    s[:, _TOK] = -1.0
    sd["pos_queries"] = torch.stack([s, -s], dim=-1).reshape(1, L, D).float().contiguous()
    E = torch.zeros_like(sd["text_embed.embedding.weight"])
    rs = math.sqrt(D)
    m = marked(torch.arange(E.shape[0]))
    E[m, 2 * _TOK] = 2.0 / rs
    E[m, 2 * _TOK + 1] = -2.0 / rs
    bos = s[0].clone()
    bos[_CODE: _CODE + _NBITS] = -1.0
    E[cfg.num_tokens - 2] = torch.stack([bos, -bos], dim=-1).reshape(D) / rs
    sd["text_embed.embedding.weight"] = E


def dec_self_order(key, T=None, extra_chars=0, mll=25, seed=7) -> Probe:
    """Which keys the self-attention sees.  Context row k carries the 7-bit code of k (BOS 0) and a token indicator.
    Every layer l, three heads with queries from the bias alone:
      head 0: key k scores 64 (k - 64), so the latest visible key wins by e^-64; v = the parity of k: flips pair (l, 0)
              when the latest visible key is odd;
      head 1: the same scores, v = the token indicator of the latest visible key (the image's own id there): pair (l, 1);
      head 2: key k scores -64 (k + 1), the earliest visible key (BOS) wins and the running max never moves; v = 1 on
              even keys: pair (l, 2);
      head 3 (layers l >= 1): head 0's scores, v = 1 where the key's content row kept pair (l - 1, 0) unflipped in
              layer l - 1, i.e. where the latest key that content row saw under the content mask was even: pair (l, 3).
              So a content mask off by one key moves the output at depth >= 2.
    A mask that lets a later key through or hides the latest one (a causal leak, a dropped own key, a padding mask
    starting one late or hiding only EOS keys, a cloze mask on the wrong key) moves the latest visible key, and an
    extra zero key (score 0) takes every head's weight.  Ids and first EOS differ per image, so a read of another
    image's ids, table rows or cache rows flips head 1."""
    cfg, sd, over = _decoder_base(key, seed, 1.0, T, extra_chars, mll)
    D, h = cfg.embed_dim, cfg.dec_num_heads
    d = D // h
    rs = math.sqrt(d)
    L, C = cfg.max_label_length + 1, cfg.num_classes
    _self_rows(sd, cfg)
    top = 32 * (2 ** _NBITS - 1)                             # sum of the code weights 32 * 2^j
    for l in range(cfg.dec_depth):
        p = f"decoder.layers.{l}.self_attn."
        W, b = sd[p + "in_proj_weight"], sd[p + "in_proj_bias"]
        for hd, sign, offset in ((0, 1.0, 32.0), (1, 1.0, 32.0), (2, -1.0, top + 64.0)):
            o = hd * d
            for j in range(_NBITS):
                b[o + j] = sign * 32.0 * 2 ** j * rs         # score = sum_j 32 * 2^j * (+-1) - offset
                W[D + o + j, 2 * (_CODE + j)] = 1.0
            b[o + _NBITS] = -offset * rs
            b[D + o + _NBITS] = 1.0
        W[2 * D: 2 * D + d, 2 * _CODE], b[2 * D: 2 * D + d] = 0.5, 0.5                  # parity
        W[2 * D + d: 2 * D + 2 * d, 2 * _TOK], b[2 * D + d: 2 * D + 2 * d] = 0.5, 0.5    # token indicator
        W[2 * D + 2 * d: 2 * D + 3 * d, 2 * _CODE], b[2 * D + 2 * d: 2 * D + 3 * d] = -0.5, 0.5   # even
        heads = 3
        if l >= 1:                                           # head 3: the content stream's own result of layer l - 1
            heads = 4
            o = 3 * d
            for j in range(_NBITS):
                b[o + j] = 32.0 * 2 ** j * rs
                W[D + o + j, 2 * (_CODE + j)] = 1.0
            b[o + _NBITS] = -32.0 * rs
            b[D + o + _NBITS] = 1.0
            W[2 * D + o: 2 * D + o + d, 2 * _flip_pair(l - 1, 0)], b[2 * D + o: 2 * D + o + d] = 0.5, 0.5
        Wo = sd[p + "out_proj.weight"]
        for hd in range(heads):
            r = 2 * _flip_pair(l, hd)
            Wo[r, hd * d: (hd + 1) * d] = -2.0 / d           # (+1, -1) + 2 v (-1, +1): flips when v = 1
            Wo[r + 1, hd * d: (hd + 1) * d] = 2.0 / d
    ctx = self_context(SELF_B, L, C, cfg.num_tokens - 2, SELF_EOS[26 if L <= 32 else 64], 300 + seed)
    bugs = {"self_extra_zero_key": _AR + _REFINE + _NAR, "self_mask_leak": _AR + _REFINE, "self_drop_own_key": _AR,
            "cloze_mask_shift": _REFINE, "eos_mask_off_by_one": _REFINE, "eos_mask_eos_only": _REFINE}
    return _dec_probe("dec_self_order", key, cfg, sd, [(bug, key) for bug in bugs], 1e-4, over, seed, B=SELF_B,
                      ctx=ctx, moves=bugs)


def dec_self_query(key, T=None, extra_chars=0, mll=25, seed=8) -> Probe:
    """The self-attention's LayerNorms and query precision.  The query stream and the context rows at amplitude delta
    (row variance ~ 2e-5), where eps 1e-6 instead of 1e-5 raises the LayerNorm gain from 0.81 to 0.98; BOS's row has
    the key indicator (pair 0) at -1, every other context row at +1.  Every layer l:
      head 0: the query reads norm_q's gain through the shared pattern and scores every key but BOS 113 or more below
              BOS at the right gain, above it at the bug's; v = (norm_c's key indicator + 0.8125) / 2, which is 0 on BOS
              at norm_c's right gain only: adds 2^-4 sum(v) to pair (l, 0);
      head 1: q = (1 + 2^-9, -1, 1) against keys -2^14 (s, s) and 16 s of the indicator s: BOS scores 13 and the others
              -13: q's bits below bf16 carry 2^14 * 2^-9 = 32 of the dot product with each key's indicator, 26 at
              gain 0.8125, which decides the sign; a bf16 q lets the others win by 26.  Same v and output, on pair
              (l, 1).
    With a single key (NAR, AR query 0) only norm_c's gain is seen, through v."""
    cfg, sd, over = _decoder_base(key, seed, 1.0, T, extra_chars, mll)
    eps, eps_bug = 1e-5, 1e-6
    dl, A, Ab = _ln_amplitude(eps, eps_bug)
    D, h = cfg.embed_dim, cfg.dec_num_heads
    d = D // h
    rs = math.sqrt(d)
    s = sd["pos_queries"][0, 0].clone()
    s[: 2 * (_TIED + 1)] = 0.0
    sd["pos_queries"] = (dl * sd["pos_queries"]).float()
    E = torch.zeros_like(sd["text_embed.embedding.weight"])
    bos = sd["pos_queries"][0, 0].clone()
    bos[2 * _KEY], bos[2 * _KEY + 1] = -dl, dl
    E[cfg.num_tokens - 2] = bos / math.sqrt(D)
    sd["text_embed.embedding.weight"] = E
    Ah, Abh = float(_bf(A)), float(_bf(Ab))
    mid = (Ah + Abh) / 2
    ns = float(s.abs().sum())
    kappa = 64.0
    for l in range(cfg.dec_depth):
        p = f"decoder.layers.{l}.self_attn."
        W, b = sd[p + "in_proj_weight"], sd[p + "in_proj_bias"]
        # q_0 (scaled) = g (gain_q - mid) < 0; k_0 = kappa gain_c s_key: the other keys score q_0 * 2 kappa gain_c
        # against BOS, at least 120 below it at the right gains and 120 above it at norm_q's bug
        g = 120.0 / (2 * kappa * Ah) / min(mid - Ah, Abh - mid)
        w = float(_bf(g * rs / ns))
        W[0] = w * s
        b[0] = -w * ns * mid
        W[D, 2 * _KEY] = kappa
        b[d], b[d + 1], b[d + 2] = (1 + 2.0 ** -9) * rs, -1.0 * rs, 1.0 * rs
        W[D + d, 2 * _KEY], W[D + d + 1, 2 * _KEY], W[D + d + 2, 2 * _KEY] = -2.0 ** 14, -2.0 ** 14, 16.0
        W[2 * D: 2 * D + 2 * d, 2 * _KEY], b[2 * D: 2 * D + 2 * d] = 0.5, 0.5 * Ah
        Wo = sd[p + "out_proj.weight"]
        Wo[2 * _flip_pair(l, 0), :d] = 2.0 ** -4
        Wo[2 * _flip_pair(l, 1), d: 2 * d] = 2.0 ** -4
    L, C = cfg.max_label_length + 1, cfg.num_classes
    ctx = self_context(SELF_B, L, C, cfg.num_tokens - 2, SELF_EOS[26 if L <= 32 else 64], 400 + seed)
    bugs = {"norm_qc_eps": _AR + _REFINE + _NAR, "self_q_bf16": _AR + _REFINE}
    return _dec_probe("dec_self_query", key, cfg, sd, [(bug, key) for bug in bugs], 1e-4, over, seed, B=SELF_B,
                      ctx=ctx, moves=bugs)


def _kname(key):
    return f"{'D' if isinstance(key[0], int) else ''}{key[0]}-depth{key[1]}"


ENCODER_KEYS = [(192, 1), (192, 2), (384, 1), (384, 2), (768, 1), (768, 2), ("vitstr", 2), ("vitstr-tail", 2)]
DECODER_KEYS = [(192, 1), (384, 1), (768, 1), (384, 2)]
WIDE_EXTRA = 100                # 195 head classes: the cluster kernel's class-sliced head
# T = 32, 65, 130 and 240 put key T inside a K/V box (zero-filled rows past the last key); at 256 the last key ends the
# last box, where a dropped last key, not an extra one, is what could go wrong
CROSS_T = (32, 65, 130, 240, 256)
SELF_KINDS = (dec_self_order, dec_self_query)
DEC_KINDS = (dec_cross, dec_ln_eps) + SELF_KINDS


def all_probes():
    """Every probe of the separation test: (builder, arguments)."""
    out = []
    for key in ENCODER_KEYS:
        out += [(enc_attention, (key,)), (enc_gelu, (key,)), (enc_ln_eps, (key,))]
        if key[0] in ("vitstr", "vitstr-tail"):
            out.append((vitstr_rounding, (key,)))
    for key in DECODER_KEYS:
        out += [(fn, (key,)) for fn in DEC_KINDS]
        out += [(fn, (key, None, 0, 63)) for fn in SELF_KINDS if key[1] > 1]    # depth 2 at L = 64
    for D in (192, 384, 768):                   # the class-sliced head (195 classes) and ids pitch 64 (L = 64)
        for extra, mll in ((WIDE_EXTRA, 25), (0, 63), (WIDE_EXTRA, 63)):
            out += [(fn, ((D, 1), None, extra, mll)) for fn in DEC_KINDS]
    for T in CROSS_T:
        out.append((dec_cross, ((384, 1), T)))
    return out
