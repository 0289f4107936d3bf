"""ctypes binding of libgoslam_b200.so.

The C header include/goslam_b200.h is the one statement of the ABI: load() parses its prototypes and sets every
entry's restype / argtypes from them.  Entries that return an int status are called through `call`, which passes
tensors as device pointers, adds the current stream and raises on an error code.

No CPU fallback lives here or anywhere else in the product path: if the shared library is missing it is built with
nvcc (go-slam_b200/build.py); if a kernel cannot launch the caller gets a RuntimeError.
"""
import ctypes
import os
import re
import threading

import torch

from . import build as _build

_lock = threading.Lock()
_LIB = None
HEADER = os.path.join(_build.ROOT, "include", "goslam_b200.h")
SIGNATURES = {}            # name -> (restype, argtypes) of every function the header declares, filled by load()
_TAKES_STREAM = set()      # names whose last parameter is `void* stream`
_ws_cache = {}

c_void_p, c_int, c_float, c_size_t, c_int64 = (
    ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t, ctypes.c_int64)


class NeusParams(ctypes.Structure):
    _fields_ = [
        ("grid", c_void_p), ("sdf_w", c_void_p), ("sdf_b", c_void_p), ("color_B", c_void_p),
        ("mlp_w", c_void_p), ("bound", c_float * 6), ("rt_bound", c_float * 6),
        ("inv_s", c_float), ("cos_anneal_ratio", c_float),
    ]


class NeusOut(ctypes.Structure):
    _fields_ = [
        ("color", c_void_p), ("depth", c_void_p), ("depth_variance", c_void_p),
        ("normal", c_void_p), ("weight_sum", c_void_p), ("sdf", c_void_p), ("z_mid", c_void_p),
        ("gradient_error", c_void_p), ("alpha", c_void_p), ("grad", c_void_p), ("pos", c_void_p),
        ("rgb", c_void_p), ("mlp_in", c_void_p), ("enc", c_void_p), ("fallback", c_void_p),
    ]


class NeusMlpBwdOut(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("H1", "H2", "dH1", "dH2", "dY8", "dE", "d_out", "h", "pts_hl", "d_grad_total")]


class BaPeers(ctypes.Structure):
    _fields_ = [("world", c_int), ("rank", c_int), ("system", c_void_p * 8), ("disps", c_void_p * 8), ("flags", c_void_p * 8),
                ("epoch", ctypes.c_uint), ("timeout", c_void_p)]


class GruWeights(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("w_zr", "w_q", "w_w", "b_zr", "b_q", "b_w", "w_glo", "b_glo")]


class UpdateWeights(ctypes.Structure):
    _fields_ = [("gru", GruWeights)] + [(n, c_void_p) for n in (
        "corr0_w", "corr0_b", "corr2_w", "corr2_b", "flow0_w", "flow0_b", "flow2_w", "flow2_b", "hid_w", "hid_b",
        "delta_w", "delta_b", "weight_w", "weight_b", "agg1_w", "agg1_b", "agg2_w", "agg2_b", "eta_w", "eta_b",
        "upmask_w", "upmask_b")]


class ConvDesc(ctypes.Structure):
    _fields_ = [("inp", c_void_p * 4), ("cin", c_int * 4), ("cin_off", c_int * 4), ("cin_stride", c_int * 4), ("n_in", c_int),
                ("weight", c_void_p), ("bias", c_void_p), ("taps", c_int), ("cout", c_int), ("cout_pad", c_int), ("act", c_int),
                ("out_scale", c_float), ("out", c_void_p), ("out_f32", c_int), ("out_stride", c_int), ("out_offset", c_int),
                ("split", c_int), ("act2", c_int), ("out2", c_void_p)]


class EncoderConv(ctypes.Structure):
    _fields_ = [("w", c_void_p), ("b", c_void_p)]


class EncoderWeights(ctypes.Structure):
    _fields_ = [("stem", EncoderConv), ("block", (EncoderConv * 3) * 6), ("out", EncoderConv)]


# C struct name -> its Structure above; a pointer to one binds as ctypes.POINTER of it
STRUCTS = {"goslam_neus_params": NeusParams, "goslam_neus_out": NeusOut, "goslam_neus_mlp_bwd_out": NeusMlpBwdOut,
           "goslam_ba_peers": BaPeers, "goslam_gru_weights": GruWeights, "goslam_update_weights": UpdateWeights,
           "goslam_conv_desc": ConvDesc, "goslam_encoder_conv": EncoderConv, "goslam_encoder_weights": EncoderWeights}

_SCALARS = {"void": None, "int": c_int, "unsigned": ctypes.c_uint, "float": c_float, "double": ctypes.c_double,
            "size_t": c_size_t, "int64_t": c_int64, "long long": c_int64}


def _ctype(decl, proto):
    """the ctypes type of a C type without a name ('const float* ', 'int64_t', ...)"""
    stars = decl.count("*")
    base = " ".join(w for w in decl.replace("*", " ").split() if w != "const")
    if stars == 0 and base in _SCALARS:
        return _SCALARS[base]
    if stars == 1 and base == "char":
        return ctypes.c_char_p
    if stars == 1 and base in STRUCTS:
        return ctypes.POINTER(STRUCTS[base])
    if stars > 0 and base:
        return c_void_p
    raise ValueError("%s: no ctypes binding for the C type %r" % (proto, decl.strip()))


def parse_header(text):
    """name -> (restype, argtypes, takes_stream) of every goslam_* prototype in the header text; takes_stream: the last
    parameter is `void* stream`"""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^[ \t]*#[^\n]*", " ", text, flags=re.M)
    text = re.sub(r"\btypedef\s+struct\b[^{;]*\{.*?\}\s*\w+\s*;", " ", text, flags=re.S)
    sigs = {}
    for ret, name, params in re.findall(r"([\w\s*]+?)\b(goslam_\w+)\s*\(([^()]*)\)\s*;", text):
        decls = [p.strip() for p in params.split(",")]
        if decls == ["void"]:
            decls = []
        argtypes = []
        for d in decls:
            m = re.fullmatch(r"(.*?)\b[A-Za-z_]\w*", d, flags=re.S)      # the type, without the parameter name
            argtypes.append(_ctype(m.group(1) if m else d, name))
        stream = bool(decls) and re.sub(r"\s+", "", decls[-1]) == "void*stream"
        sigs[name] = (_ctype(ret, name), argtypes, stream)
    return sigs


def lib_path():
    return _build.LIB


def load(build_if_missing=True):
    """Return the loaded CDLL (building it first if the .so is absent), bound as the header declares it."""
    global _LIB
    with _lock:
        if _LIB is not None:
            return _LIB
        path = lib_path()
        if not os.path.exists(path):
            if not build_if_missing:
                raise RuntimeError("libgoslam_b200.so not built (run python -m __graft_entry__ or "
                                   "go-slam_b200/build.py)")
            _build.build()
        with open(HEADER) as f:
            sigs = parse_header(f.read())
        lib = ctypes.CDLL(path)
        for name, (res, args, stream) in sigs.items():
            fn = getattr(lib, name)          # AttributeError => header/library mismatch
            fn.restype = res
            fn.argtypes = args
            SIGNATURES[name] = (res, args)
            if stream:
                _TAKES_STREAM.add(name)
        _LIB = lib
        return lib


def check(rc, what):
    if rc != 0:
        msg = load().goslam_strerror(int(rc))
        detail = load().goslam_last_cuda_error() if int(rc) == -2 else b""
        raise RuntimeError("%s failed: %s (code %d)%s" % (what, msg.decode() if msg else "?", rc,
                                                          ": " + detail.decode() if detail else ""))


def call(name, *args, device=None):
    """goslam_<name>(*args) for an entry that returns an int status.  A tensor goes as its device pointer (a CPU tensor
    raises), None as NULL, anything else (ctypes objects, ints, floats) as it is.  Runs on `device`, else on the device
    of the first tensor, else on the current device, and appends that device's current stream when the prototype ends
    in `void* stream`; raises RuntimeError on a non-zero status.  It neither synchronises, allocates nor queries the
    device, so it may run inside a CUDA graph capture.  The tensors stay referenced until the launch has been issued."""
    fname = "goslam_" + name
    fn = getattr(_LIB or load(), fname)
    conv = list(args)
    dev = device
    for i, a in enumerate(conv):
        if isinstance(a, torch.Tensor):
            if not a.is_cuda:
                raise RuntimeError("%s: tensors must live on a CUDA device (there is no CPU fallback)" % fname)
            if dev is None:
                dev = a.device
            conv[i] = a.data_ptr()
    with torch.cuda.device(dev):
        if fname in _TAKES_STREAM:
            conv.append(torch.cuda.current_stream().cuda_stream)
        rc = fn(*conv)
    check(rc, name)


def workspace(nbytes, device):
    """grow-only per-device scratch (borrowed for the duration of one call on the current stream)."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


def need_cuda(what, *ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("%s: tensors must live on a CUDA device (there is no CPU fallback)" % what)


def contig(**kw):
    for name, t in kw.items():
        if not t.is_contiguous():
            raise RuntimeError("%s must be contiguous" % name)


def ptr_array(tensors):
    """host array of the tensors' device pointers (the library's `const void* const*` parameters)"""
    need_cuda("ptr_array", *tensors)
    arr = (ctypes.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


def ptr(t):
    """device pointer of a torch tensor (or None)."""
    return None if t is None else c_void_p(t.data_ptr())


def stream_ptr():
    return c_void_p(torch.cuda.current_stream().cuda_stream)
