"""When does `engine()` upload the weights again?  (No GPU.)

A model keeps one engine handle for its lifetime and uploads its parameters to it only when they changed
(_EngineModule.engine).  Here a recording stand-in replaces the engine: it keeps a copy of every state_dict it is sent.
For every way of changing the weights - load_state_dict strict or partial, with assign=True, inside or outside
inference mode, on inference-tensor parameters, through the ViTSTR and PARSeq systems' own load_state_dict, a replaced
parameter, an optimizer step and `.to()` - the next engine() call must upload exactly the model's new weights, and a
second call with nothing changed in between must upload nothing (the check stays cheap: no upload per call).

A compiled Lexicon holds class ids of one charset and words of at most one max_label_length: a model with another
charset of the same size, or another max_label_length, must refuse it."""
import functools

import pytest
import torch
from torch import nn

import parseq_b200.system as S
from parseq_b200.factory import create_model
from parseq_b200.weights import init_state_dict


class RecordingEngine:
    """Stands in for parseq_b200.engine.Engine: records every state_dict it is sent."""

    def __init__(self, cfg, device):
        self.cfg, self.device, self.loads = cfg, device, []

    def set_option(self, name, value):
        pass

    def load_state_dict(self, sd, stream):
        self.loads.append({k: v.detach().to(torch.float32).clone() for k, v in sd.items()})


@pytest.fixture(autouse=True)
def stand_in(monkeypatch):
    monkeypatch.setattr(S, "Engine", RecordingEngine)
    monkeypatch.setattr(S._EngineModule, "_device", property(lambda self: torch.device("cuda", 0)))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: type("Stream", (), {"cuda_stream": 0})())


def _create(arch, **kw):
    """parseq-tiny, or ViTSTR at parseq-tiny's width (the weight plumbing does not depend on the width)."""
    if arch == "parseq":
        return create_model("parseq-tiny", **kw)
    return create_model("vitstr", embed_dim=192, enc_num_heads=3, **kw)


@functools.lru_cache(maxsize=None)
def _init(arch, seed):
    return init_state_dict(_create(arch).model.cfg, seed)


def _sd(arch, seed):
    """A fresh copy: load_state_dict(assign=True) makes these tensors the parameters."""
    return {k: v.clone() for k, v in _init(arch, seed).items()}


def _system(arch, inference=False):
    """A parseq-tiny or ViTSTR system (built inside inference mode: inference-tensor parameters) on seed 0."""
    with torch.inference_mode(inference):
        m = _create(arch)
        m.model.load_state_dict(_sd(arch, 0))
    return m


def _expect_upload(model, want):
    """engine() uploads `want` (key -> tensor) once, and a second call uploads nothing."""
    eng = model.engine()
    n = len(eng.loads)
    assert n >= 1, "no upload"
    got = eng.loads[-1]
    assert set(got) == set(want)
    bad = [k for k in want if not torch.equal(got[k], want[k].to(torch.float32))]
    assert not bad, f"the engine holds stale values of {bad[:4]}"
    assert model.engine() is eng and len(eng.loads) == n, "an engine() call with no change uploaded the weights"


def _current(model):
    return {k: v.detach() for k, v in model.state_dict().items()}


def _reload(m, sd, **kw):
    m.model.load_state_dict(sd, **kw)


def _reload_inference(m, sd, **kw):
    with torch.inference_mode():
        m.model.load_state_dict(sd, **kw)


def _partial(m, sd):
    m.model.load_state_dict({k: v for k, v in sd.items() if k.startswith("head.")}, strict=False)


def _system_prefixed(m, sd, **kw):
    m.load_state_dict({"model." + k: v for k, v in sd.items()}, **kw)


def _replace_parameter(m, sd):
    m.model.head.weight = nn.Parameter(sd["head.weight"].clone(), requires_grad=False)
    m.model.head.bias = nn.Parameter(sd["head.bias"].clone(), requires_grad=False)


def _replace_root_parameter(m, sd):
    name = "pos_queries" if "pos_queries" in sd else "pos_embed"
    setattr(m.model, name, nn.Parameter(sd[name].clone(), requires_grad=False))


def _optimizer_step(m, sd):
    """One SGD step that lands every parameter on `sd` (p -= 1 * (p - sd[k]))."""
    params = dict(m.model.named_parameters())
    for k, p in params.items():
        p.grad = p.detach() - sd[k]
    torch.optim.SGD(params.values(), lr=1.0).step()


# name -> (how the weights change, which weights the engine must then hold: "new" = the seed-1 state_dict, "head" =
# seed 0 with seed 1's head, "model" = whatever the model's parameters now are)
CHANGES = {
    "load_state_dict": (_reload, "new"),
    "load_state_dict_partial": (_partial, "head"),
    "load_state_dict_assign": (lambda m, sd: _reload(m, sd, assign=True), "new"),
    "load_state_dict_in_inference_mode": (_reload_inference, "new"),
    "load_state_dict_assign_in_inference_mode": (lambda m, sd: _reload_inference(m, sd, assign=True), "new"),
    "system_load_state_dict": (_system_prefixed, "new"),
    "system_load_state_dict_assign": (lambda m, sd: _system_prefixed(m, sd, assign=True), "new"),
    "replace_parameter": (_replace_parameter, "head"),
    "replace_root_parameter": (_replace_root_parameter, "model"),
    "optimizer_step": (_optimizer_step, "model"),
    "to_float64": (lambda m, sd: m.to(torch.float64), "model"),
}


def _want(m, kind, sd0, sd1):
    if kind == "new":
        return sd1
    if kind == "head":
        return {k: (sd1[k] if k.startswith("head.") else sd0[k]) for k in sd0}
    return _current(m.model)


@pytest.mark.parametrize("arch", ["parseq", "vitstr"])
@pytest.mark.parametrize("change", sorted(CHANGES))
def test_next_engine_call_uploads_the_new_weights(arch, change):
    m = _system(arch)
    sd0, sd1 = _sd(arch, 0), _sd(arch, 1)
    _expect_upload(m.model, sd0)
    fn, kind = CHANGES[change]
    fn(m, sd1)
    _expect_upload(m.model, _want(m, kind, sd0, sd1))
    if kind != "model":                    # and back: the engine follows every change, not only the first
        fn(m, sd0)
        _expect_upload(m.model, sd0)


@pytest.mark.parametrize("arch", ["parseq", "vitstr"])
@pytest.mark.parametrize("assign", [False, True], ids=["copy", "assign"])
def test_inference_tensor_parameters_reloaded(arch, assign):
    """A model built and loaded under inference_mode has inference-tensor parameters: no version counter, and an
    in-place reload keeps every parameter's identity."""
    m = _system(arch, inference=True)
    assert m.model.head.bias.is_inference()
    sd0, sd1 = _sd(arch, 0), _sd(arch, 1)
    _expect_upload(m.model, sd0)
    _reload_inference(m, sd1, assign=assign)
    _expect_upload(m.model, sd1)
    _reload_inference(m, sd0, assign=assign)
    _expect_upload(m.model, sd0)


def test_vitstr_system_load_state_dict_accepts_both_layouts():
    m = _system("vitstr", inference=True)
    sd0, sd1 = _sd("vitstr", 0), _sd("vitstr", 1)
    _expect_upload(m.model, sd0)
    with torch.inference_mode():
        m.load_state_dict({"model." + k: v for k, v in sd1.items()})
    _expect_upload(m.model, sd1)
    with torch.inference_mode():
        m.load_state_dict(sd0)
    _expect_upload(m.model, sd0)


def test_no_change_no_upload():
    m = _system("parseq")
    eng = m.model.engine()
    assert len(eng.loads) == 1
    for _ in range(3):
        m.model.engine()
    m.model.set_engine_option("chunk", 64)
    m.model.engine()
    m.model.state_dict()                    # reading the weights changes nothing
    m.model.engine()
    assert len(eng.loads) == 1


def _charset_of_same_size(cs):
    """`cs` with its first two characters swapped: the same class count, different class ids."""
    return cs[1] + cs[0] + cs[2:]


@pytest.mark.parametrize("arch", ["parseq", "vitstr"])
@pytest.mark.parametrize("size", ["same_size", "one_more"])
def test_lexicon_of_another_charset_refused(arch, size):
    m = _system(arch)
    cs = m.model.cfg.charset_train
    other = _create(arch, charset_train=_charset_of_same_size(cs) if size == "same_size" else cs + "\u00e9")
    assert (other.model.cfg.num_classes == m.model.cfg.num_classes) == (size == "same_size")
    words = [cs[:3], cs[1] + cs[5]]
    lex = other.compile_lexicon(words)
    x = torch.zeros((1, 3, *m.model.cfg.img_size))
    with pytest.raises(ValueError, match="charset"):
        m.beam_search(x, 2, lexicon=lex)
    with pytest.raises(ValueError, match="charset"):
        m.lexicon_decode(x, lex, beam_width=2)
    with pytest.raises(ValueError, match="charset"):
        m.model.beam_search(x, 2, lexicon=lex)
    assert m.model._engine is None, "a refused lexicon reached the engine"


@pytest.mark.parametrize("arch", ["parseq", "vitstr"])
@pytest.mark.parametrize("other_length", [40, 10])
def test_lexicon_of_another_max_label_length_refused(arch, other_length):
    m = _system(arch)
    cs = m.model.cfg.charset_train
    other = _create(arch, max_label_length=other_length)
    lex = other.compile_lexicon([cs[:3], cs[4:9]])
    x = torch.zeros((1, 3, *m.model.cfg.img_size))
    with pytest.raises(ValueError, match="max_label_length"):
        m.beam_search(x, 2, lexicon=lex)
    assert m.model._engine is None, "a refused lexicon reached the engine"


def test_lexicon_of_the_same_model_passes_the_checks():
    """The model's own lexicon gets past the host checks (it then needs CUDA images: the stand-in has no device)."""
    m = _system("parseq")
    cs = m.model.cfg.charset_train
    lex = m.compile_lexicon([cs[:3], cs[4:9]])
    x = torch.zeros((1, 3, *m.model.cfg.img_size))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.beam_search(x, 2, lexicon=lex)
