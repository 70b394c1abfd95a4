"""GPU: every device buffer, stream, event and graph exec an engine or a lexicon allocates is released.

The engine's resource owners keep two process-wide counts, read through parseq_debug_int(NULL, "live_device_bytes") and
parseq_debug_int(NULL, "live_cuda_objects") (streams, events, graph execs).  A handle taken through every kind of
call returns both to where they were before it was created; a lexicon returns its arrays whether it goes before or
after its engine; a resize leaves what a handle created at the final sizes holds after the same calls; graphs dropped
by an option change or a weight reload and recaptured leave both counts where they were."""
import gc

import pytest
import torch

from test_gpu_handle_lifetime import _cfg_sd, _float, _u8, build, catalogue, release, run

pytestmark = pytest.mark.gpu


def counters():
    """(live device bytes, live CUDA objects), with the collected handles released and the device idle."""
    from parseq_b200.engine import load_library
    lib = load_library()
    gc.collect()
    torch.cuda.synchronize()
    return int(lib.parseq_debug_int(None, b"live_device_bytes")), int(lib.parseq_debug_int(None, b"live_cuda_objects"))


# forwards through the float, uint8, device-crops, host and host-crops entry points (two super-chunks included),
# attention maps (PARSeq), score, beam search, and lexicon beam search with a shared and a per-image lexicon
PARSEQ_CALLS = ("fwd_float_b300", "fwd_u8_b5", "fwd_crops_b4", "fwd_host_float_b3", "fwd_host_u8_b6",
                "fwd_host_crops_big_b3", "fwd_b700", "maps_b5", "maps_ar0_b4", "score_many", "beam_k8", "lex_large",
                "lex_per_image_large")
VITSTR_CALLS = ("fwd_float_b300", "fwd_u8_b5", "fwd_host_float_b4", "fwd_host_crops_big_b3", "fwd_b700", "score_many",
                "beam_k8", "lex_large", "lex_per_image_large")


def calls_of(kind, names=None):
    cat = dict(catalogue(kind))
    return [(n, cat[n]) for n in (names or (VITSTR_CALLS if kind == "vitstr" else PARSEQ_CALLS))]


def run_all(m, calls):
    for _, call in calls:
        run(m, call)


@pytest.mark.parametrize("kind", ["s95", "s195", "d2", "vitstr"])
def test_a_handle_returns_everything(kind):
    """Graph and eager calls of every kind; s195: above 128 classes (the top-K epilogue's beam buffers), d2: decoder
    depth 2 (per-layer content K/V caches)."""
    base = counters()
    m = build(kind)
    for graph in (1, 0):
        m.model.set_engine_option("use_graph", graph)
        run_all(m, calls_of(kind))
    used = counters()
    assert used[0] > base[0] and used[1] > base[1]
    release(m)
    del m
    assert counters() == base, f"{kind}: (bytes, objects) {used} while alive, not back to {base} after destroy"


@pytest.mark.parametrize("order", ["lexicon_first", "engine_first"])
def test_a_lexicon_releases_its_arrays(order):
    base = counters()
    m = build("s95")
    run_all(m, calls_of("s95", ["lex_large"]))     # the engine's lexicon buffers, so that only the lexicon's own count
    cs = m.model.cfg.charset_train
    lex = m.compile_lexicon([cs[i % 50:i % 50 + 1 + i % 7] for i in range(40)])
    x = _float(_u8(m.model.cfg, 3, 60)).cuda()
    without = counters()
    with torch.inference_mode():
        m.beam_search(x, 4, lexicon=lex)           # shared: no roots to upload
    with_lex = counters()
    assert with_lex == (without[0] + lex.nbytes, without[1])
    if order == "lexicon_first":
        del lex
        assert counters() == without
        release(m)
    else:
        release(m)
        assert counters() == (base[0] + lex.nbytes, base[1])
        del lex
    del m
    assert counters() == base


def test_resize_up_then_down_holds_what_a_fresh_handle_holds():
    """max_batch, chunk and dec_chunk up, then down, each followed by the calls that reserve on-demand buffers (maps,
    scoring, beam and lexicon buffers, the host-crop staging buffer): the handle then holds exactly what a handle
    created at the final sizes holds after the same calls."""
    calls = calls_of("s95", ["fwd_float_b300", "fwd_host_crops_big_b3", "maps_b5", "score_many", "beam_k8", "lex_large",
                             "lex_per_image_large"])
    steps = [("chunk", 128), ("dec_chunk", 32),                                # from max_batch 512, chunk 512, dec_chunk 128
             ("max_batch", 1024), ("chunk", 512), ("dec_chunk", 256),         # up
             ("max_batch", 384), ("chunk", 96), ("dec_chunk", 48)]            # down
    final = [("max_batch", 384), ("chunk", 96), ("dec_chunk", 48)]
    base = counters()
    m = build("s95")
    run_all(m, calls)
    for opt, value in steps:
        m.model.set_engine_option(opt, value)
        run_all(m, calls)
    resized = counters()
    resized_beam = m.model.engine().debug_int("beam_bytes")
    release(m)
    del m
    assert counters() == base
    f = build("s95", options=final)
    run_all(f, calls)
    fresh = counters()
    fresh_beam = f.model.engine().debug_int("beam_bytes")
    release(f)
    del f
    assert counters() == base
    assert resized[0] - base[0] == fresh[0] - base[0], (resized, fresh, base)
    assert resized_beam == fresh_beam
    assert resized[1] - base[1] == fresh[1] - base[1]


@pytest.mark.parametrize("kind", ["s95", "d2"])
def test_dropped_graphs_are_released_when_recaptured(kind):
    """Option changes that drop the graphs, and weight reloads: once the same calls have run again (graphs
    recaptured), the handle holds the same bytes and CUDA objects as before."""
    calls = calls_of(kind, ["fwd_float_b300", "fwd_float_b3", "fwd_host_u8_b6", "maps_b5", "score_few", "beam_k2"])
    m = build(kind)
    run_all(m, calls)
    want = counters()
    _, sd1 = _cfg_sd(kind, 1)
    _, sd0 = _cfg_sd(kind, 0)
    changes = [("pdl", 0), ("pdl", 1), ("fuse_ln", 0), ("fuse_ln", 3), ("ar_kernel", 0), ("ar_kernel", 2),
               ("ar_cluster_size", 6), ("ar_cluster_size", 0), ("weights", sd1), ("weights", sd0)]
    bad = []
    for name, value in changes:
        if name == "weights":
            m.model.load_state_dict(value)
            name = "reload"
        else:
            m.model.set_engine_option(name, value)
        run_all(m, calls)
        got = counters()
        if got != want:
            bad.append(f"{name}: {got} != {want}")
    release(m)
    assert not bad, bad
