"""GPU: what each engine call launches.

`parseq_kernel_launches` counts every kernel an engine call enqueues (a CUDA graph counts the kernels it was captured
with).  The counts below pin, per kind of call, how many kernels one call launches: forward on every entry point and
schedule (graph and eager), the host split pipeline, several decoder chains, every AR loop; score, beam search and
lexicon beam search at depth 1 and 2, at <= 128 and > 128 head classes and on ViTSTR; and the decoder module API.  The
host code that drives these calls can be restructured freely, but a change to what it launches shows up here."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SCHEDULES = {"ar_refine": (True, 1), "nar": (False, 1), "ar_maps": (True, 0)}
ENTRIES = ("float", "u8", "crops", "host_float", "host_u8", "host_crops")

# parseq_kernel_launches of one call, as the engine launched them when this test was written (PARSeq-S / ViTSTR-S with
# 12 encoder blocks, max_label_length 25)
PINNED = {
    "c195/beam_k1": 389, "c195/beam_k4": 389, "c195/forward": 94, "c195/lexicon_k4": 389,
    "c195/lexicon_per_image_k2": 389, "c195/score": 89, "chunks4/beam_k1": 937, "chunks4/beam_k4": 3520,
    "chunks4/forward_b12": 122, "chunks4/lexicon_k4": 3520, "chunks4/lexicon_per_image_k2": 1798, "chunks4/score": 141,
    "d2/beam_k1": 1039, "d2/beam_k4": 1039, "d2/forward": 1029, "d2/forward_maps": 1022, "d2/lexicon_k4": 1039,
    "d2/lexicon_per_image_k2": 1039, "d2/score": 115, "decode_ex": 13, "encode": 75, "forward/eager/ar_maps/crops": 88,
    "forward/eager/ar_maps/float": 87, "forward/eager/ar_maps/host_crops": 88, "forward/eager/ar_maps/host_float": 87,
    "forward/eager/ar_maps/host_u8": 87, "forward/eager/ar_maps/u8": 87, "forward/eager/ar_refine/crops": 95,
    "forward/eager/ar_refine/float": 94, "forward/eager/ar_refine/host_crops": 95,
    "forward/eager/ar_refine/host_float": 94, "forward/eager/ar_refine/host_u8": 94, "forward/eager/ar_refine/u8": 94,
    "forward/eager/nar/crops": 104, "forward/eager/nar/float": 103, "forward/eager/nar/host_crops": 104,
    "forward/eager/nar/host_float": 103, "forward/eager/nar/host_u8": 103, "forward/eager/nar/u8": 103,
    "forward/graph/ar_maps/crops": 88, "forward/graph/ar_maps/float": 87, "forward/graph/ar_maps/float_ar_kernel0": 346,
    "forward/graph/ar_maps/float_ar_kernel1": 87, "forward/graph/ar_maps/host_crops": 88,
    "forward/graph/ar_maps/host_float": 87, "forward/graph/ar_maps/host_u8": 87, "forward/graph/ar_maps/u8": 87,
    "forward/graph/ar_refine/crops": 95, "forward/graph/ar_refine/float": 94,
    "forward/graph/ar_refine/float_ar_kernel0": 353, "forward/graph/ar_refine/float_ar_kernel1": 94,
    "forward/graph/ar_refine/float_b300": 98, "forward/graph/ar_refine/float_b300_maps": 101,
    "forward/graph/ar_refine/host_crops": 95, "forward/graph/ar_refine/host_float": 94,
    "forward/graph/ar_refine/host_float_b256": 183, "forward/graph/ar_refine/host_u8": 94,
    "forward/graph/ar_refine/u8": 94, "forward/graph/nar/crops": 104, "forward/graph/nar/float": 103,
    "forward/graph/nar/host_crops": 104, "forward/graph/nar/host_float": 103, "forward/graph/nar/host_u8": 103,
    "forward/graph/nar/u8": 103, "head": 2, "s/beam_k1": 363, "s/beam_k4": 363, "s/lexicon_k4": 363,
    "s/lexicon_per_image_k2": 363, "s/score": 89, "vitstr/beam_k1": 117, "vitstr/beam_k4": 117,
    "vitstr/forward/float": 92, "vitstr/forward/host_float": 92, "vitstr/lexicon_k4": 117,
    "vitstr/lexicon_per_image_k2": 117, "vitstr/score": 91, "vitstr_c195/beam_k1": 117, "vitstr_c195/beam_k4": 117,
    "vitstr_c195/lexicon_k4": 117, "vitstr_c195/lexicon_per_image_k2": 117, "vitstr_c195/score": 91,
}


def _model(experiment="parseq", n_extra=0, dec_depth=1):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    extra = {} if experiment == "vitstr" else {"dec_depth": dec_depth}
    cfg = make_config_long(experiment, 25, n_extra, **extra)
    m = create_model(experiment, charset_train=charset(n_extra), max_label_length=25, **extra)
    m.model.load_state_dict(init_state_dict(cfg, 0))
    return cfg, m.eval().to("cuda")


def _counted(m, fn):
    eng = m.model.engine()
    torch.cuda.synchronize()
    before = eng.launches
    with torch.inference_mode():
        fn()
    torch.cuda.synchronize()
    return eng.launches - before


def _images(cfg, B, seed):
    from parseq_b200.weights import synth_images
    return synth_images(cfg, B, seed).cuda()


def _forward(m, cfg, entry, B, sched, maps=False):
    """Launches of one forward call through `entry` (the low-level entry points, as parseq_forward* take them)."""
    from parseq_b200.system import _crops_c, pack_crops
    eng = m.model.engine()
    ar, refine = SCHEDULES[sched]
    maps = maps or sched == "ar_maps"
    host = entry.startswith("host")
    dev = torch.device("cpu") if host else torch.device("cuda")
    g = torch.Generator().manual_seed(B)
    H, W = cfg.img_size
    u8 = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    x = u8.permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5).contiguous()
    crops = [torch.randint(0, 256, (20 + 7 * (i % 5), 60 + 13 * (i % 7), 3), generator=g, dtype=torch.uint8)
             for i in range(B)]
    L = eng.num_steps(None)
    logits = torch.empty((B, L, cfg.num_classes), dtype=torch.float32, device=dev, pin_memory=host)
    ids = torch.empty((B, L), dtype=torch.int32, device=dev, pin_memory=host)
    steps = torch.empty((1,), dtype=torch.int32, device=dev, pin_memory=host)
    amap = torch.empty((B, L, cfg.num_patches), dtype=torch.float32, device=dev, pin_memory=host) if maps else None
    kw = {"attn_maps_ptr": amap.data_ptr()} if maps else {}
    st = torch.cuda.current_stream().cuda_stream
    ptrs = (logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), st, None, ar, refine)
    if entry == "float":
        xs = x.cuda()
        return _counted(m, lambda: eng.forward(xs.data_ptr(), B, *ptrs, **kw))
    if entry == "host_float":
        xs = x.pin_memory()
        return _counted(m, lambda: eng.forward_host(xs.data_ptr(), B, *ptrs, **kw))
    if entry in ("u8", "host_u8"):
        us = u8.pin_memory() if host else u8.cuda()
        return _counted(m, lambda: eng.forward_u8(us.data_ptr(), B, *ptrs, host=host, **kw))
    data, offsets, sizes = pack_crops(crops, pin_memory=True) if host else pack_crops([c.cuda() for c in crops])
    return _counted(m, lambda: eng.forward_crops(_crops_c(data, offsets, sizes, 0), B, *ptrs, host=host, **kw))


def _candidates(cs, N, per, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(N):
        row = []
        for _ in range(per):
            n = int(torch.randint(1, 10, (1,), generator=g))
            row.append("".join(cs[int(i)] for i in torch.randint(0, len(cs), (n,), generator=g)))
        out.append(row)
    return out


def _words(cs, k, seed):
    return [w for row in _candidates(cs, 1, k, seed) for w in row]


def _decoders(m, cfg, tag, out, N=6):
    """score, beam search and lexicon beam search of N images."""
    cs = cfg.charset_train
    x = _images(cfg, N, 7)
    out[f"{tag}/score"] = _counted(m, lambda: m.score(x, _candidates(cs, N, 4, 1)))
    for K in (1, 4):
        out[f"{tag}/beam_k{K}"] = _counted(m, lambda: m.beam_search(x, K))
    words = _words(cs, 12, 2)
    out[f"{tag}/lexicon_k4"] = _counted(m, lambda: m.beam_search(x, 4, lexicon=words))
    per = [_words(cs, 3, 10 + b) for b in range(N)]
    out[f"{tag}/lexicon_per_image_k2"] = _counted(m, lambda: m.beam_search(x, 2, lexicon=per))


def measure_parseq():
    out = {}
    cfg, m = _model()
    for mode, graph in (("graph", 1), ("eager", 0)):
        m.model.set_engine_option("use_graph", graph)
        for sched in SCHEDULES:
            for entry in ENTRIES:
                out[f"forward/{mode}/{sched}/{entry}"] = _forward(m, cfg, entry, 3, sched)
    m.model.set_engine_option("use_graph", 1)
    # the host pipeline's two halves (>= 256 images), and three decoder chains with and without maps
    out["forward/graph/ar_refine/host_float_b256"] = _forward(m, cfg, "host_float", 256, "ar_refine")
    out["forward/graph/ar_refine/float_b300"] = _forward(m, cfg, "float", 300, "ar_refine")
    out["forward/graph/ar_refine/float_b300_maps"] = _forward(m, cfg, "float", 300, "ar_refine", maps=True)
    for k in (0, 1):
        m.model.set_engine_option("ar_kernel", k)
        for sched in ("ar_refine", "ar_maps"):
            out[f"forward/graph/{sched}/float_ar_kernel{k}"] = _forward(m, cfg, "float", 3, sched)
    m.model.set_engine_option("ar_kernel", 2)
    _decoders(m, cfg, "s", out)
    # decoder module API (parseq_encode, parseq_decode_ex, parseq_head)
    x = _images(cfg, 5, 3)
    tgt = torch.randint(1, 95, (5, 8))
    tgt[:, 0] = cfg.num_tokens - 2
    tgt = tgt.cuda()
    mem = {}
    out["encode"] = _counted(m, lambda: mem.setdefault("m", m.model.encode(x)))
    out["decode_ex"] = _counted(m, lambda: mem.setdefault("y", m.model.decode(tgt, mem["m"])))
    out["head"] = _counted(m, lambda: m.model.head(mem["y"]))
    # many small decoder chains: forward, score and beam groups spread round-robin over the stages
    for k, v in (("max_batch", 16), ("dec_chunk", 4)):
        m.model.set_engine_option(k, v)
    out["chunks4/forward_b12"] = _forward(m, cfg, "float", 12, "ar_refine")
    _decoders(m, cfg, "chunks4", out, N=12)
    return out


def measure_others():
    out = {}
    cfg, m = _model(dec_depth=2)
    out["d2/forward"] = _forward(m, cfg, "float", 3, "ar_refine")
    out["d2/forward_maps"] = _forward(m, cfg, "float", 3, "ar_maps")
    _decoders(m, cfg, "d2", out)
    cfg, m = _model(n_extra=100)              # 195 head classes: the top-K epilogue and the lexicon's logits rows
    out["c195/forward"] = _forward(m, cfg, "float", 3, "ar_refine")
    _decoders(m, cfg, "c195", out)
    cfg, m = _model("vitstr")
    for entry in ("float", "host_float"):
        out[f"vitstr/forward/{entry}"] = _forward(m, cfg, entry, 3, "nar")
    _decoders(m, cfg, "vitstr", out)
    cfg, m = _model("vitstr", n_extra=100)
    _decoders(m, cfg, "vitstr_c195", out)
    return out


@pytest.mark.parametrize("measure", [measure_parseq, measure_others], ids=["parseq", "others"])
def test_launches_per_call(measure):
    got = measure()
    print(got)
    want = {k: v for k, v in PINNED.items() if k in got}
    assert set(want) == set(got), sorted(set(got) ^ set(want))
    assert got == want, {k: (got[k], want[k]) for k in got if got[k] != want[k]}
