"""The C-ABI library loads and exports every symbol include/*.h declares (no compute, no GPU)."""
import ctypes
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header):
    src = open(header).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sv[a-z]*_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def built():
    from sceneverse_b200 import build
    build.build_all()
    return build


@pytest.mark.parametrize("header", sorted(glob.glob(os.path.join(ROOT, "include", "*.h"))))
def test_header_symbols_exported(built, header):
    names = _declared(header)
    assert names, header
    libname = {"svpointops.h": "libsvpointops.so", "svgps.h": "libsvgps.so"}[os.path.basename(header)]
    lib = ctypes.CDLL(os.path.join(built.LIBDIR, libname))
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, f"{libname} does not export {missing}"


def test_status_strings_and_arg_checks(built):
    from sceneverse_b200 import _lib
    lib = _lib.pointops()
    assert lib.sv_version() >= 100
    assert lib.sv_status_string(0) == b"ok"
    # argument validation happens before any CUDA call
    assert lib.sv_fps_f32(None, 1, 0, 1, None, None, None) == 1
    assert lib.sv_fps_f32(None, 0, 16, 4, None, None, None) == 0  # empty batch is a no-op
    assert lib.sv_ball_query_f32(None, None, 1, 8, 4, 0.2, 600, None, None) == 1
    assert lib.sv_fps_ballquery_f32(None, 1, 2048, 4, 0.2, 8, None, None, None, None) == 1


def test_ext_rejects_cpu_and_bad_dtypes(built):
    import torch
    from sceneverse_b200.pointnet2 import _ext
    with pytest.raises(RuntimeError, match="CPU not supported"):
        _ext.furthest_point_sampling(torch.zeros(1, 8, 3), 2)
    with pytest.raises(RuntimeError, match="float tensor"):
        _ext.furthest_point_sampling(torch.zeros(1, 8, 3, dtype=torch.float64), 2)
    with pytest.raises(RuntimeError, match="contiguous"):
        _ext.gather_points(torch.zeros(1, 8, 3).transpose(1, 2), torch.zeros(1, 2, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="int tensor"):
        _ext.gather_points(torch.zeros(1, 3, 8), torch.zeros(1, 2, dtype=torch.int64))


def test_dropin_import_name(built):
    import sys
    from sceneverse_b200 import dropin
    ext = dropin.install()
    import pointnet2._ext as _ext  # the reference's import statement (pointnet2_utils.py:23)
    assert _ext is ext
    for fn in ["gather_points", "gather_points_grad", "furthest_point_sampling", "three_nn", "three_interpolate",
               "three_interpolate_grad", "ball_query", "group_points", "group_points_grad"]:  # bindings.cpp:6-19
        assert callable(getattr(_ext, fn))
    sys.modules.pop("pointnet2", None)
    sys.modules.pop("pointnet2._ext", None)


def test_gps_argument_validation_without_gpu(built):
    """libsvgps rejects malformed calls before touching the device (status 1 = SV_ERR_INVALID_ARG, 0 for empty work)."""
    from sceneverse_b200 import _lib
    lib = _lib.gps()
    fake = 0x1000  # 16-byte aligned, never dereferenced: validation fails first
    # transposed A needs lda >= M and lda % 8 == 0; K-major operands need K % 8 == 0
    assert lib.sv_gemm_bf16_ex(fake, 777, 1, fake, 320, 1, 777, 320, 1000, None, 0, None, fake, 320, 1, 0, None) == 1
    assert lib.sv_gemm_bf16_ex(fake, 130, 0, fake, 2048, 1, 64, 2048, 130, None, 0, None, fake, 2048, 1, 0, None) == 1
    assert lib.sv_gemm_bf16_ex(fake, 64, 0, fake, 64, 0, 0, 64, 64, None, 0, None, fake, 64, 0, 0, None) == 0
    assert lib.sv_layer_norm_fwd(fake, None, 1, 4, 770, fake, fake, 1e-5, 0.0, 0, fake, None, fake, fake, None) == 1   # D % 8
    assert lib.sv_layer_norm_fwd(fake, fake, 1, 4, 768, fake, fake, 1e-5, 0.0, 0, fake, None, fake, fake, None) == 1  # residual needs s
    assert lib.sv_colsum(fake, 100, 1, 4, 100, fake, fake, None) == 1                                                # N % 8
    assert lib.sv_attention_fwd_dropout_bf16(fake, 8, 8, fake, 8, 8, fake, 8, 8, fake, 8, 8, None, None, 0, None, 1, 12, 4,
                                             400, 0.125, None, 0.0, 0, None) == 1                                      # Lk > 384
    assert lib.sv_layer_norm_scratch_floats(768) > 0 and lib.sv_colsum_scratch_floats(768) > 0


def test_argtypes_bound_from_headers(built):
    """After loading, every prototype of both headers has argtypes, one per parameter the header declares."""
    from sceneverse_b200 import _lib
    for header, lib in (("svpointops.h", _lib.pointops()), ("svgps.h", _lib.gps())):
        src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", header)).read(), flags=re.S)
        protos = re.findall(r"\b(sv\w*)\s*\(([^()]*)\)\s*;", src)
        assert len(protos) > 10, header
        for name, params in protos:
            n_params = 0 if params.strip() == "void" else params.count(",") + 1
            argtypes = getattr(lib, name).argtypes
            assert argtypes is not None and len(argtypes) == n_params, (header, name, argtypes)


def test_header_types_pinned(built):
    from sceneverse_b200 import _lib
    pointops, gps = _lib.pointops(), _lib.gps()
    assert pointops.sv_scene_prep_aug_f32.argtypes[5] is ctypes.POINTER(_lib.AugParams)
    fwd = gps.sv_attention_fwd_dropout_bf16.argtypes
    assert fwd[22] is ctypes.c_float and fwd[23] is ctypes.c_ulonglong   # dropout_p, seed
    assert pointops.sv_status_string.restype is ctypes.c_char_p
    assert pointops.sv_launch_count.restype is ctypes.c_ulonglong
    assert gps.svgps_launch_count.restype is ctypes.c_ulonglong


@pytest.mark.parametrize("proto", ["int sv_x(size_t n, void *stream);", "size_t sv_x(int n);"])
def test_unknown_header_type_raises(proto):
    from sceneverse_b200 import _lib
    with pytest.raises(_lib.NativeLibraryError, match="sv_x"):
        _lib.parse_prototypes(proto)
