"""ctypes binding of libsvpointops and libsvgps.  Argument and return types come from the headers the libraries are built
against (include/svpointops.h, include/svgps.h).  No fallback: if the CUDA library is missing or a call fails this raises —
the product path never routes around the native code."""
import ctypes
import os
import re

import torch

_LIBDIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib")
_INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
_cache = {}

c_int, c_float, c_void_p = ctypes.c_int, ctypes.c_float, ctypes.c_void_p

# include/svpointops.h sv_aug_params
AUG_FLIP, AUG_SCALE, AUG_SCENE_TRANS, AUG_SCENE_ROT, AUG_COLOR = 1, 2, 4, 8, 16
AUG_OBJ_TRANS, AUG_OBJ_ROT, AUG_JITTER, AUG_PTS_SHUFFLE = 32, 64, 128, 256
AUG_ITEM_STRIDE, AUG_OBJ_STRIDE = 25, 12


# include/svgps.h evaluation counter layouts (float64 words)
EVAL_GROUNDING, EVAL_OBJ_CLS, EVAL_ANSWERS, EVAL_PRETRAIN = 0, 1, 2, 3
(EVG_ITEMS, EVG_MULTIPLE, EVG_HARD, EVG_VIEW_DEP, EVG_OG_ACC, EVG_OG_ACC_HARD, EVG_OG_ACC_VIEW_DEP, EVG_IOU25, EVG_IOU50,
 EVG_IOU25_MULTIPLE, EVG_IOU50_MULTIPLE, EVG_TXT_ACC, EVG_OBJ) = range(13)
EVG_SIZE = EVG_OBJ + 6
EVO_HIT, EVO_COUNT, EVO_SIZE = 0, 1, 2
EVA_NTYPES = 6
EVA_ITEMS, EVA_ANS1, EVA_ANS10, EVA_TYPE_ITEMS, EVA_TYPE_ANS1, EVA_OBJ_HIT, EVA_OBJ_COUNT = 0, 1, 2, 3, 9, 15, 16
EVA_SNAPSHOT, EVA_Q_ANS1, EVA_Q_ANS10, EVA_Q_OBJ, EVA_Q_TYPE, EVA_Q_TYPE_COUNT, EVA_SIZE = 17, 34, 35, 36, 37, 43, 49
EVP_OG, EVP_ITEMS, EVP_LM_HIT, EVP_LM_COUNT, EVP_OBJ, EVP_SNAPSHOT, EVP_Q, EVP_SIZE = 0, 12, 13, 14, 15, 33, 66, 76
(EVP_Q_TARGET, EVP_Q_OG, EVP_Q_LM, EVP_Q_POST, EVP_Q_PRE, EVP_Q_RAW, EVP_Q_PRE_UNMASK, EVP_Q_PRE_MASK, EVP_Q_POST_UNMASK,
 EVP_Q_POST_MASK) = range(10)
EVP_HAS_OG, EVP_HAS_POST, EVP_HAS_RAW, EVP_HAS_PRE = 1, 2, 4, 8
TRAIN_LOG_MAX_VALUES = 32


class AugParams(ctypes.Structure):
    _fields_ = [("flags", c_int), ("scene_rot_axis_align", c_int), ("scene_rot_shuffle", c_int),
                ("obj_rot_axis_align", c_int), ("obj_rot_shuffle", c_int),
                ("scale_lo", ctypes.c_double), ("scale_hi", ctypes.c_double),
                ("scene_trans", ctypes.c_double * 3), ("scene_rot", ctypes.c_double * 3),
                ("obj_trans", ctypes.c_double * 3), ("obj_rot", ctypes.c_double * 3), ("jitter", ctypes.c_double)]


class NativeLibraryError(RuntimeError):
    pass


def _load(name):
    if name in _cache:
        return _cache[name]
    path = os.path.join(_LIBDIR, name)
    if not os.path.exists(path):
        raise NativeLibraryError(
            f"{path} is missing: build it with `python -m sceneverse_b200.build` "
            "(sceneverse_b200 has no CPU or PyTorch fallback)")
    lib = ctypes.CDLL(path)
    _cache[name] = lib
    return lib


# C type -> ctypes type of every non-pointer parameter and return type the headers use; any other type is an error
_CTYPES = {"int": c_int, "unsigned": ctypes.c_uint, "float": c_float, "double": ctypes.c_double,
           "long long": ctypes.c_longlong, "unsigned long long": ctypes.c_ulonglong}
_PROTOTYPE = re.compile(r"([\w\s*]+?)\b(\w+)\s*\(([^()]*)\)")
_PARAM = re.compile(r"([\w\s*]*?)\s*\b(\w+)")


def _ctype(decl, fn, is_return):
    """The ctypes type of one C declaration without its name ("const float *", "unsigned long long")."""
    base = " ".join(w for w in decl.replace("*", " ").split() if w != "const")
    if "*" in decl:
        if base == "sv_aug_params" and not is_return:
            return ctypes.POINTER(AugParams)
        if base == "char" and is_return:
            return ctypes.c_char_p
        return c_void_p
    if base in _CTYPES:
        return _CTYPES[base]
    raise NativeLibraryError(f"{fn}: no ctypes mapping for the C type '{decl.strip()}'")


def parse_prototypes(text):
    """{name: (restype, argtypes)} of every prototype `ret name(params);` of a C header, after comments, preprocessor lines
    and `extern "C" {` are stripped.  Statements without parentheses (typedefs, enums) are skipped."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^[ \t]*#[^\n]*", " ", text, flags=re.M)
    text = re.sub(r'extern\s+"C"\s*\{', " ", text)
    protos = {}
    for stmt in text.split(";"):
        if "(" not in stmt:
            continue
        m = _PROTOTYPE.fullmatch(stmt.strip())
        if m is None:
            raise NativeLibraryError(f"not a prototype: '{' '.join(stmt.split())}'")
        ret, name, params = m.groups()
        argtypes = []
        if params.strip() != "void":
            for param in params.split(","):
                pm = _PARAM.fullmatch(param.strip())
                if pm is None:
                    raise NativeLibraryError(f"{name}: cannot parse the parameter '{' '.join(param.split())}'")
                argtypes.append(_ctype(pm.group(1), name, False))
        protos[name] = (_ctype(ret, name, True), argtypes)
    return protos


def _bind(lib, header):
    """Sets argtypes / restype of every function `header` (include/) declares."""
    with open(os.path.join(_INCLUDE, header)) as f:
        protos = parse_prototypes(f.read())
    for name, (restype, argtypes) in protos.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes


def pointops():
    lib = _load("libsvpointops.so")
    if not getattr(lib, "_sv_ready", False):
        _bind(lib, "svpointops.h")
        lib._sv_ready = True
    return lib


def gps():
    lib = _load("libsvgps.so")
    if not getattr(lib, "_sv_ready", False):
        _bind(lib, "svgps.h")
        # status strings live in libsvpointops
        lib.sv_status_string = pointops().sv_status_string
        lib.sv_last_cuda_error_string = lib.svgps_last_cuda_error_string
        lib._sv_ready = True
    return lib


def ptr(t):
    """The device pointer of tensor `t`, or NULL for None."""
    return None if t is None else t.data_ptr()


def call(lib, name, device, *args):
    """lib.name(*args, stream) under `device`, with that device's current stream appended; raises if the status is not 0."""
    with torch.cuda.device(device):
        st = getattr(lib, name)(*args, torch.cuda.current_stream(device).cuda_stream)
    check(lib, st, name)


def check(lib, status, what):
    if status != 0:
        msg = lib.sv_status_string(status).decode()
        if status == 2:
            msg += ": " + lib.sv_last_cuda_error_string().decode()
        raise RuntimeError(f"{what} failed: {msg}")


def launch_count():
    """Kernel launches enqueued so far by both native libraries."""
    n = int(pointops().sv_launch_count())
    import os as _os
    if _os.path.exists(_os.path.join(_LIBDIR, "libsvgps.so")):
        n += int(gps().svgps_launch_count())
    return n
