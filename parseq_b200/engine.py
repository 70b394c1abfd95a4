"""ctypes binding of include/parseq_b200.h.  The library is the product; this file only marshals
pointers.  There is no fallback: if the shared library is missing or no sm_90 device exists,
construction raises."""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional

from .build import LIB_PATH

_lib = None


class ParseqConfigC(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "img_h", "img_w", "patch_h", "patch_w", "embed_dim", "enc_num_heads", "enc_mlp_ratio", "enc_depth",
        "dec_num_heads", "dec_mlp_ratio", "dec_depth", "max_label_length", "num_tokens", "max_batch", "device", "arch")]


class ForwardArgsC(C.Structure):
    _fields_ = [("batch", C.c_int32), ("max_length", C.c_int32), ("decode_ar", C.c_int32),
                ("refine_iters", C.c_int32), ("forced_ids", C.c_void_p), ("forced_refine", C.c_void_p),
                ("class_mask", C.c_void_p), ("attn_maps", C.c_void_p)]


class CropsC(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_bytes", C.c_int64), ("offsets", C.c_void_p), ("sizes", C.c_void_p),
                ("rotation", C.c_int32), ("rotations", C.c_void_p)]


class RegionsC(C.Structure):
    _fields_ = [("frames", C.c_void_p), ("frames_bytes", C.c_int64), ("frame_offsets", C.c_void_p),
                ("frame_sizes", C.c_void_p), ("num_frames", C.c_int32), ("frame_index", C.c_void_p), ("sizes", C.c_void_p),
                ("coeffs", C.c_void_p)]


class PolygonsC(C.Structure):
    _fields_ = [("frames", C.c_void_p), ("frames_bytes", C.c_int64), ("frame_offsets", C.c_void_p),
                ("frame_sizes", C.c_void_p), ("num_frames", C.c_int32), ("frame_index", C.c_void_p), ("sizes", C.c_void_p),
                ("num_points", C.c_void_p), ("points", C.c_void_p)]


class OrientArgsC(C.Structure):
    _fields_ = [("num_orientations", C.c_int32), ("orientations", C.c_int32 * 4), ("min_confidence", C.c_float),
                ("rotation_out", C.c_void_p), ("confidence_out", C.c_void_p)]


def orient_args(orientations, min_confidence, rotation_ptr, confidence_ptr) -> OrientArgsC:
    """parseq_orient_args: up to four orientations, min_confidence None for none (NaN)."""
    o = list(orientations)
    return OrientArgsC(len(o), (C.c_int32 * 4)(*(o + [0] * (4 - len(o)))[:4]),
                       float("nan") if min_confidence is None else float(min_confidence), rotation_ptr, confidence_ptr)


class ScoreArgsC(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_candidates", C.c_int32), ("per_image", C.c_void_p), ("targets", C.c_void_p),
                ("lengths", C.c_void_p), ("attn_maps", C.c_void_p)]


class BeamArgsC(C.Structure):
    _fields_ = [("batch", C.c_int32), ("beam_width", C.c_int32), ("max_length", C.c_int32), ("class_mask", C.c_void_p),
                ("attn_maps", C.c_void_p)]


class LexiconDescC(C.Structure):
    _fields_ = [("num_nodes", C.c_int32), ("num_edges", C.c_int32), ("first_edge", C.c_void_p), ("edge_class", C.c_void_p),
                ("edge_child", C.c_void_p), ("terminal", C.c_void_p)]


class BeamSelectArgsC(C.Structure):
    _fields_ = [("logits", C.c_void_p), ("part", C.c_void_p), ("keys", C.c_void_p), ("ntiles", C.c_int32),
                ("row0", C.c_int64), ("img_stride", C.c_int64), ("slot_stride", C.c_int64),
                ("batch", C.c_int32), ("num_classes", C.c_int32), ("beam_width", C.c_int32), ("step", C.c_int32),
                ("num_steps", C.c_int32), ("class_mask", C.c_void_p), ("mask_ld", C.c_int32),
                ("ids_in", C.c_void_p), ("score_in", C.c_void_p), ("len_in", C.c_void_p), ("st_in", C.c_void_p),
                ("ids_out", C.c_void_p), ("score_out", C.c_void_p), ("len_out", C.c_void_p), ("st_out", C.c_void_p),
                ("parent", C.c_void_p), ("ids_ld", C.c_int32), ("out_ids", C.c_void_p), ("out_len", C.c_void_p),
                ("out_score", C.c_void_p), ("first_edge", C.c_void_p), ("edge_class", C.c_void_p),
                ("edge_child", C.c_void_p), ("terminal", C.c_void_p), ("roots", C.c_void_p), ("node_in", C.c_void_p),
                ("node_out", C.c_void_p)]


def lexicon_desc(first_edge, edge_class, edge_child, terminal) -> LexiconDescC:
    """parseq_lexicon_desc over contiguous numpy arrays (int32, int32, int32, uint8); the caller keeps them alive."""
    return LexiconDescC(int(terminal.shape[0]), int(edge_class.shape[0]), first_edge.ctypes.data, edge_class.ctypes.data,
                        edge_child.ctypes.data, terminal.ctypes.data)


class LexiconHandle:
    """Owns one `parseq_lexicon*` (a lexicon on one device)."""

    def __init__(self, lib, ptr):
        self.lib, self.ptr = lib, ptr

    def __del__(self):
        try:
            if self.ptr:
                self.lib.parseq_lexicon_destroy(self.ptr)
                self.ptr = None
        except Exception:
            pass


EXPORTS = [
    "parseq_create", "parseq_destroy", "parseq_set_weight", "parseq_num_weights", "parseq_weight_key",
    "parseq_finalize", "parseq_forward", "parseq_forward_host", "parseq_forward_u8", "parseq_forward_host_u8",
    "parseq_resize_crops", "parseq_warp_regions", "parseq_tps_coeffs", "parseq_warp_polygons",
    "parseq_forward_crops", "parseq_forward_host_crops", "parseq_forward_crops_oriented",
    "parseq_score", "parseq_score_u8", "parseq_score_check", "parseq_beam_search", "parseq_beam_search_u8",
    "parseq_lexicon_check", "parseq_lexicon_create", "parseq_lexicon_destroy", "parseq_beam_search_lexicon",
    "parseq_beam_search_lexicon_u8",
    "parseq_postprocess", "parseq_encode", "parseq_decode", "parseq_decode_ex", "parseq_head", "parseq_text_embed", "parseq_kernel_launches", "parseq_debug_int", "parseq_bench_tma_stream",
    "parseq_set_option", "parseq_get_timing", "parseq_get_ar_profile", "parseq_last_error", "parseq_version", "parseq_gemm_bf16", "parseq_gemm_ln_bf16", "parseq_mlp_ln_bf16", "parseq_layernorm_bf16",
    "parseq_enc_attention", "parseq_qkv_attention_bf16", "parseq_head_lse_bf16", "parseq_head_topk_bf16",
    "parseq_beam_select",
]


def load_library(path: Optional[str] = None):
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or os.environ.get("PARSEQ_B200_LIB", LIB_PATH)
    if not os.path.exists(p):
        raise RuntimeError(f"{p} not found: build it with `python -m parseq_b200.build` "
                           "(there is no CPU / PyTorch fallback)")
    lib = C.CDLL(p)
    lib.parseq_last_error.restype = C.c_char_p
    lib.parseq_version.restype = C.c_char_p
    lib.parseq_weight_key.restype = C.c_char_p
    lib.parseq_weight_key.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int64)]
    lib.parseq_bench_tma_stream.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.parseq_debug_int.restype = C.c_int64
    lib.parseq_debug_int.argtypes = [C.c_void_p, C.c_char_p]
    lib.parseq_kernel_launches.restype = C.c_int64
    lib.parseq_kernel_launches.argtypes = [C.c_void_p]
    lib.parseq_create.argtypes = [C.POINTER(ParseqConfigC), C.POINTER(C.c_void_p)]
    lib.parseq_destroy.argtypes = [C.c_void_p]
    lib.parseq_destroy.restype = None
    lib.parseq_set_weight.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]
    lib.parseq_num_weights.argtypes = [C.c_void_p]
    lib.parseq_finalize.argtypes = [C.c_void_p, C.c_void_p]
    lib.parseq_forward.argtypes = [C.c_void_p, C.POINTER(ForwardArgsC), C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p]
    lib.parseq_forward_host.argtypes = lib.parseq_forward.argtypes
    lib.parseq_forward_u8.argtypes = lib.parseq_forward.argtypes
    lib.parseq_forward_host_u8.argtypes = lib.parseq_forward.argtypes
    lib.parseq_resize_crops.argtypes = [C.c_void_p, C.c_int32, C.POINTER(CropsC), C.c_void_p, C.c_void_p]
    lib.parseq_warp_regions.argtypes = [C.c_void_p, C.c_int32, C.POINTER(RegionsC), C.c_void_p, C.c_int64, C.c_void_p]
    lib.parseq_tps_coeffs.argtypes = [C.c_int32, C.c_void_p, C.c_void_p]
    lib.parseq_warp_polygons.argtypes = [C.c_void_p, C.c_int32, C.POINTER(PolygonsC), C.c_void_p, C.c_int64, C.c_void_p]
    lib.parseq_forward_crops.argtypes = [C.c_void_p, C.POINTER(ForwardArgsC), C.POINTER(CropsC), C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p]
    lib.parseq_forward_host_crops.argtypes = lib.parseq_forward_crops.argtypes
    lib.parseq_forward_crops_oriented.argtypes = [C.c_void_p, C.POINTER(ForwardArgsC), C.POINTER(CropsC),
                                                  C.POINTER(OrientArgsC), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_score.argtypes = [C.c_void_p, C.POINTER(ScoreArgsC), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_score_u8.argtypes = lib.parseq_score.argtypes
    lib.parseq_score_check.argtypes = [C.POINTER(ParseqConfigC), C.POINTER(ScoreArgsC)]
    lib.parseq_beam_search.argtypes = [C.c_void_p, C.POINTER(BeamArgsC), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    lib.parseq_beam_search_u8.argtypes = lib.parseq_beam_search.argtypes
    lib.parseq_lexicon_check.argtypes = [C.POINTER(ParseqConfigC), C.POINTER(LexiconDescC)]
    lib.parseq_lexicon_create.argtypes = [C.c_void_p, C.POINTER(LexiconDescC), C.POINTER(C.c_void_p), C.c_void_p]
    lib.parseq_lexicon_destroy.argtypes = [C.c_void_p]
    lib.parseq_lexicon_destroy.restype = None
    lib.parseq_beam_search_lexicon.argtypes = [C.c_void_p, C.POINTER(BeamArgsC), C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_beam_search_lexicon_u8.argtypes = lib.parseq_beam_search_lexicon.argtypes
    lib.parseq_postprocess.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p]
    lib.parseq_encode.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_decode.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_decode_ex.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_head.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_text_embed.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int64]
    lib.parseq_get_timing.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                      C.POINTER(C.c_int64)]
    lib.parseq_gemm_bf16.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int,
                                     C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                     C.c_int64, C.c_void_p]
    lib.parseq_gemm_ln_bf16.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]
    lib.parseq_mlp_ln_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]
    lib.parseq_layernorm_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_int,
                                          C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_enc_attention.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.parseq_qkv_attention_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                              C.c_void_p, C.c_void_p]
    lib.parseq_head_lse_bf16.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_head_topk_bf16.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                          C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.parseq_beam_select.argtypes = [C.POINTER(BeamSelectArgsC), C.c_void_p]
    if path is None:
        _lib = lib
    return lib


class EngineError(RuntimeError):
    pass


def check(lib, rc: int):
    if rc != 0:
        raise EngineError(f"parseq_b200 error {rc}: {lib.parseq_last_error().decode()}")


def tps_coeffs(points, lib=None):
    """parseq_tps_coeffs: the TPS coefficients T float64 [F + 3, 2] of F polygon points [F, 2] in engine order (top edge,
    then bottom edge, each left to right).  Needs the library, not a device."""
    import numpy as np
    lib = lib or load_library()
    p = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 2)
    t = np.empty((len(p) + 3, 2), dtype=np.float64)
    check(lib, lib.parseq_tps_coeffs(len(p), p.ctypes.data, t.ctypes.data))
    return t


def config_c(cfg, device: int = 0, max_batch: int = 0) -> ParseqConfigC:
    return ParseqConfigC(cfg.img_size[0], cfg.img_size[1], cfg.patch_size[0], cfg.patch_size[1], cfg.embed_dim,
                         cfg.enc_num_heads, cfg.enc_mlp_ratio, cfg.enc_depth, cfg.dec_num_heads, cfg.dec_mlp_ratio,
                         cfg.dec_depth, cfg.max_label_length, cfg.num_tokens, max_batch, device,
                         1 if getattr(cfg, "arch", "parseq") == "vitstr" else 0)


class Engine:
    """Owns one `parseq_engine*`."""

    def __init__(self, cfg, device: int = 0, max_batch: int = 0):
        self.lib = load_library()
        self.cfg = cfg
        c = config_c(cfg, device, max_batch)
        h = C.c_void_p()
        check(self.lib, self.lib.parseq_create(C.byref(c), C.byref(h)))
        self.handle = h
        self.device = device

    def close(self):
        if getattr(self, "handle", None):
            self.lib.parseq_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def weight_keys(self) -> Dict[str, int]:
        out = {}
        n = self.lib.parseq_num_weights(self.handle)
        for i in range(n):
            numel = C.c_int64()
            k = self.lib.parseq_weight_key(self.handle, i, C.byref(numel))
            out[k.decode()] = numel.value
        return out

    def load_state_dict(self, sd, stream: int = 0):
        import torch
        expected = self.weight_keys()
        missing = [k for k in expected if k not in sd]
        unexpected = [k for k in sd if k not in expected]
        if missing or unexpected:
            raise EngineError(f"state_dict mismatch: missing {missing[:4]}... unexpected {unexpected[:4]}...")
        for k, numel in expected.items():
            t = sd[k].detach().to(device="cpu", dtype=torch.float32).contiguous()
            if t.numel() != numel:
                raise EngineError(f"size mismatch for {k}: {tuple(t.shape)} vs {numel} elements")
            check(self.lib, self.lib.parseq_set_weight(self.handle, k.encode(), t.data_ptr(), numel))
        check(self.lib, self.lib.parseq_finalize(self.handle, stream))

    def set_option(self, name: str, value: int):
        check(self.lib, self.lib.parseq_set_option(self.handle, name.encode(), int(value)))

    TIMING_CATEGORIES = ("enc_gemm", "enc_attn", "layernorm", "dec_gemm", "dec_attn", "other", "enc_gemm_ln", "dec_ar",
                         "score_tail", "beam_select", "attn_maps", "orient")

    def get_timing(self):
        out = {}
        for i, name in enumerate(self.TIMING_CATEGORIES):
            ms, fl, n = C.c_double(), C.c_double(), C.c_int64()
            check(self.lib, self.lib.parseq_get_timing(self.handle, i, C.byref(ms), C.byref(fl), C.byref(n)))
            out[name] = dict(ms=ms.value, flops=fl.value, launches=n.value)
        return out

    def get_ar_profile(self):
        buf = (C.c_uint64 * 512)()
        self.lib.parseq_get_ar_profile.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        check(self.lib, self.lib.parseq_get_ar_profile(self.handle, buf))
        return [[buf[s * 16 + k] for k in range(16)] for s in range(32)]

    def debug_int(self, name: str) -> int:
        return int(self.lib.parseq_debug_int(self.handle, name.encode()))

    @property
    def launches(self) -> int:
        return int(self.lib.parseq_kernel_launches(self.handle))

    def num_steps(self, max_length) -> int:
        ml = self.cfg.max_label_length if max_length is None else min(int(max_length), self.cfg.max_label_length)
        return ml + 1

    def _args(self, batch, max_length, decode_ar, refine_iters, forced_ids=None, forced_refine=None, class_mask=None,
              attn_maps=None):
        return ForwardArgsC(batch, -1 if max_length is None else int(max_length), int(bool(decode_ar)),
                            int(refine_iters), forced_ids, forced_refine, class_mask, attn_maps)

    # class_mask_ptr: the per-image allowlist words (parseq_forward_args.class_mask), in the memory of the images;
    # attn_maps_ptr: fp32 [batch, num_steps, T] cross-attention maps (parseq_forward_args.attn_maps), in the memory of the
    # logits
    def forward(self, images_ptr, batch, logits_ptr, ids_ptr, steps_ptr, stream, max_length=None, decode_ar=True,
                refine_iters=1, forced_ids_ptr=None, forced_refine_ptr=None, class_mask_ptr=None, attn_maps_ptr=None):
        a = self._args(batch, max_length, decode_ar, refine_iters, forced_ids_ptr, forced_refine_ptr, class_mask_ptr,
                       attn_maps_ptr)
        check(self.lib, self.lib.parseq_forward(self.handle, C.byref(a), images_ptr, logits_ptr, ids_ptr, steps_ptr,
                                                stream))

    def forward_host(self, images_ptr, batch, logits_ptr, ids_ptr, steps_ptr, stream, max_length=None,
                     decode_ar=True, refine_iters=1, class_mask_ptr=None, attn_maps_ptr=None):
        a = self._args(batch, max_length, decode_ar, refine_iters, class_mask=class_mask_ptr, attn_maps=attn_maps_ptr)
        check(self.lib, self.lib.parseq_forward_host(self.handle, C.byref(a), images_ptr, logits_ptr, ids_ptr,
                                                     steps_ptr, stream))

    def forward_u8(self, images_ptr, batch, logits_ptr, ids_ptr, steps_ptr, stream, max_length=None, decode_ar=True,
                   refine_iters=1, host=False, class_mask_ptr=None, attn_maps_ptr=None):
        a = self._args(batch, max_length, decode_ar, refine_iters, class_mask=class_mask_ptr, attn_maps=attn_maps_ptr)
        fn = self.lib.parseq_forward_host_u8 if host else self.lib.parseq_forward_u8
        check(self.lib, fn(self.handle, C.byref(a), images_ptr, logits_ptr, ids_ptr, steps_ptr, stream))

    def resize_crops(self, crops: CropsC, batch, out_ptr, stream):
        check(self.lib, self.lib.parseq_resize_crops(self.handle, batch, C.byref(crops), out_ptr, stream))

    def warp_regions(self, regions: RegionsC, count, out_ptr, out_bytes, stream):
        check(self.lib, self.lib.parseq_warp_regions(self.handle, count, C.byref(regions), out_ptr, out_bytes, stream))

    def warp_polygons(self, polygons: PolygonsC, count, out_ptr, out_bytes, stream):
        check(self.lib, self.lib.parseq_warp_polygons(self.handle, count, C.byref(polygons), out_ptr, out_bytes, stream))

    def forward_crops(self, crops: CropsC, batch, logits_ptr, ids_ptr, steps_ptr, stream, max_length=None, decode_ar=True,
                      refine_iters=1, host=False, class_mask_ptr=None, attn_maps_ptr=None):
        a = self._args(batch, max_length, decode_ar, refine_iters, class_mask=class_mask_ptr, attn_maps=attn_maps_ptr)
        fn = self.lib.parseq_forward_host_crops if host else self.lib.parseq_forward_crops
        check(self.lib, fn(self.handle, C.byref(a), C.byref(crops), logits_ptr, ids_ptr, steps_ptr, stream))

    # orientation search (parseq_forward_crops_oriented): crops in device or host memory, every output on the device;
    # rotation_ptr int32 [batch] / confidence_ptr fp32 [batch] the chosen orientation and its confidence
    def forward_crops_oriented(self, crops: CropsC, batch, orientations, min_confidence, logits_ptr, ids_ptr, steps_ptr,
                               rotation_ptr, confidence_ptr, stream, max_length=None, decode_ar=True, refine_iters=1,
                               class_mask_ptr=None, attn_maps_ptr=None):
        a = self._args(batch, max_length, decode_ar, refine_iters, class_mask=class_mask_ptr, attn_maps=attn_maps_ptr)
        o = orient_args(orientations, min_confidence, rotation_ptr, confidence_ptr)
        check(self.lib, self.lib.parseq_forward_crops_oriented(self.handle, C.byref(a), C.byref(crops), C.byref(o),
                                                               logits_ptr, ids_ptr, steps_ptr, stream))

    # per_image / targets / lengths: CPU int32 tensors (parseq_score_args); scores / token_lp / attn_maps: device pointers
    def score(self, images_ptr, batch, per_image, targets, lengths, scores_ptr, token_lp_ptr, stream, u8=False,
              attn_maps_ptr=None):
        a = ScoreArgsC(batch, int(targets.shape[0]), per_image.data_ptr(), targets.data_ptr(), lengths.data_ptr(),
                       attn_maps_ptr)
        fn = self.lib.parseq_score_u8 if u8 else self.lib.parseq_score
        check(self.lib, fn(self.handle, C.byref(a), images_ptr, scores_ptr, token_lp_ptr, stream))

    # ids [N, K, num_steps] / lengths [N, K] / scores [N, K] / attn_maps [N, K, num_steps, T]: device pointers;
    # class_mask_ptr as in forward; lexicon: a LexiconHandle of this engine's device, roots a CPU int32 tensor [N] or None
    def beam_search(self, images_ptr, batch, beam_width, ids_ptr, lengths_ptr, scores_ptr, stream, max_length=None,
                    class_mask_ptr=None, u8=False, lexicon=None, roots=None, attn_maps_ptr=None):
        a = BeamArgsC(batch, int(beam_width), -1 if max_length is None else int(max_length), class_mask_ptr,
                      attn_maps_ptr)
        if lexicon is None:
            fn = self.lib.parseq_beam_search_u8 if u8 else self.lib.parseq_beam_search
            check(self.lib, fn(self.handle, C.byref(a), images_ptr, ids_ptr, lengths_ptr, scores_ptr, stream))
            return
        fn = self.lib.parseq_beam_search_lexicon_u8 if u8 else self.lib.parseq_beam_search_lexicon
        check(self.lib, fn(self.handle, C.byref(a), lexicon.ptr, roots.data_ptr() if roots is not None else None,
                           images_ptr, ids_ptr, lengths_ptr, scores_ptr, stream))

    def lexicon_create(self, first_edge, edge_class, edge_child, terminal, stream) -> LexiconHandle:
        """Uploads a lexicon (numpy CSR arrays, parseq_lexicon_desc) to this engine's device."""
        d = lexicon_desc(first_edge, edge_class, edge_child, terminal)
        h = C.c_void_p()
        check(self.lib, self.lib.parseq_lexicon_create(self.handle, C.byref(d), C.byref(h), stream))
        return LexiconHandle(self.lib, h)

    def postprocess(self, logits_ptr, batch, num_steps, ids_ptr, lengths_ptr, conf_ptr, stream, eos_id=0):
        check(self.lib, self.lib.parseq_postprocess(logits_ptr, batch, num_steps, self.cfg.num_classes, eos_id, ids_ptr,
                                                    lengths_ptr, conf_ptr, stream))

    def encode(self, images_ptr, batch, memory_ptr, stream):
        check(self.lib, self.lib.parseq_encode(self.handle, batch, images_ptr, memory_ptr, stream))

    def decode(self, batch, ctx_len, num_queries, tgt_ptr, memory_ptr, query_ptr, qmask_ptr, pmask_ptr, out_ptr, stream,
               cmask_ptr=None):
        check(self.lib, self.lib.parseq_decode_ex(self.handle, batch, ctx_len, num_queries, tgt_ptr, memory_ptr, query_ptr,
                                                  qmask_ptr, pmask_ptr, cmask_ptr, out_ptr, stream))

    def head(self, rows, x_ptr, logits_ptr, stream):
        check(self.lib, self.lib.parseq_head(self.handle, rows, x_ptr, logits_ptr, stream))

    def text_embed(self, n, ids_ptr, out_ptr, stream):
        check(self.lib, self.lib.parseq_text_embed(self.handle, n, ids_ptr, out_ptr, stream))
