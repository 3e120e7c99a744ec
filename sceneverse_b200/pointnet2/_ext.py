"""`pointnet2._ext` replacement: the nine functions of the reference's pybind module
(/root/reference/modules/third_party/pointnet2/_ext_src/src/bindings.cpp:6-19) with the same
names, argument order, dtype/contiguity preconditions (include/utils.h:5-25) and ownership rules
(fresh output tensors on the input's device; inputs never mutated), implemented by
libsvpointops (include/svpointops.h) on the current CUDA stream.

Differences by design: precondition failures raise RuntimeError (the reference AT_ASSERTs, which
also surfaces as RuntimeError); a failed launch raises instead of exit(-1)
(include/cuda_utils.h:30-39).
"""
import torch

from .. import _lib


def _check(t, name, dtype):
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous tensor")
    if t.dtype != dtype:
        raise RuntimeError(f"{name} must be a {'float' if dtype == torch.float32 else 'int'} tensor")


def _cuda_only(t, *others):
    if not t.is_cuda:
        raise RuntimeError("CPU not supported")
    for o in others:
        if not o.is_cuda:
            raise RuntimeError("must be a CUDA tensor")
        if o.device != t.device:
            raise RuntimeError("tensors must be on the same device")


def furthest_point_sampling(points, nsamples):
    """sampling.cpp:66-87.  (B,N,3) f32 -> (B,nsamples) i32."""
    _check(points, "points", torch.float32)
    _cuda_only(points)
    B, N, _ = points.shape
    out = torch.empty((B, nsamples), dtype=torch.int32, device=points.device)
    _lib.call(_lib.pointops(), "sv_fps_f32", points.device, points.data_ptr(), B, N, int(nsamples), out.data_ptr(), None)
    return out


def gather_points(points, idx):
    """sampling.cpp:15-38.  (B,C,N) f32, (B,M) i32 -> (B,C,M)."""
    _check(points, "points", torch.float32)
    _check(idx, "idx", torch.int32)
    _cuda_only(points, idx)
    B, C, N = points.shape
    M = idx.shape[1]
    out = torch.empty((B, C, M), dtype=torch.float32, device=points.device)
    _lib.call(_lib.pointops(), "sv_gather_points_f32", points.device, points.data_ptr(), idx.data_ptr(), B, C, N, M,
              out.data_ptr())
    return out


def gather_points_grad(grad_out, idx, n):
    """sampling.cpp:40-65.  (B,C,M) -> (B,C,n)."""
    _check(grad_out, "grad_out", torch.float32)
    _check(idx, "idx", torch.int32)
    _cuda_only(grad_out, idx)
    B, C, M = grad_out.shape
    out = torch.empty((B, C, int(n)), dtype=torch.float32, device=grad_out.device)
    _lib.call(_lib.pointops(), "sv_gather_points_grad_f32", grad_out.device, grad_out.data_ptr(), idx.data_ptr(), B, C, int(n),
              M, out.data_ptr())
    return out


def ball_query(new_xyz, xyz, radius, nsample):
    """ball_query.cpp:8-32.  (B,M,3), (B,N,3) -> (B,M,nsample) i32."""
    _check(new_xyz, "new_xyz", torch.float32)
    _check(xyz, "xyz", torch.float32)
    _cuda_only(new_xyz, xyz)
    B, M, _ = new_xyz.shape
    N = xyz.shape[1]
    out = torch.empty((B, M, int(nsample)), dtype=torch.int32, device=new_xyz.device)
    _lib.call(_lib.pointops(), "sv_ball_query_f32", new_xyz.device, new_xyz.data_ptr(), xyz.data_ptr(), B, N, M, float(radius),
              int(nsample), out.data_ptr())
    return out


def group_points(points, idx):
    """group_points.cpp:12-36.  (B,C,N), (B,NP,NS) i32 -> (B,C,NP,NS)."""
    _check(points, "points", torch.float32)
    _check(idx, "idx", torch.int32)
    _cuda_only(points, idx)
    B, C, N = points.shape
    _, NP, NS = idx.shape
    out = torch.empty((B, C, NP, NS), dtype=torch.float32, device=points.device)
    _lib.call(_lib.pointops(), "sv_group_points_f32", points.device, points.data_ptr(), idx.data_ptr(), B, C, N, NP, NS,
              out.data_ptr())
    return out


def group_points_grad(grad_out, idx, n):
    """group_points.cpp:38-62.  (B,C,NP,NS) -> (B,C,n)."""
    _check(grad_out, "grad_out", torch.float32)
    _check(idx, "idx", torch.int32)
    _cuda_only(grad_out, idx)
    B, C, NP, NS = grad_out.shape
    out = torch.empty((B, C, int(n)), dtype=torch.float32, device=grad_out.device)
    _lib.call(_lib.pointops(), "sv_group_points_grad_f32", grad_out.device, grad_out.data_ptr(), idx.data_ptr(), B, C, int(n),
              NP, NS, out.data_ptr())
    return out


def three_nn(unknowns, knows):
    """interpolate.cpp:14-40.  (B,n,3), (B,m,3) -> [dist2 (B,n,3) f32, idx (B,n,3) i32]."""
    _check(unknowns, "unknowns", torch.float32)
    _check(knows, "knows", torch.float32)
    _cuda_only(unknowns, knows)
    B, n, _ = unknowns.shape
    m = knows.shape[1]
    idx = torch.empty((B, n, 3), dtype=torch.int32, device=unknowns.device)
    dist2 = torch.empty((B, n, 3), dtype=torch.float32, device=unknowns.device)
    _lib.call(_lib.pointops(), "sv_three_nn_f32", unknowns.device, unknowns.data_ptr(), knows.data_ptr(), B, n, m,
              dist2.data_ptr(), idx.data_ptr())
    return [dist2, idx]


def three_interpolate(points, idx, weight):
    """interpolate.cpp:42-70.  (B,c,m), (B,n,3) i32, (B,n,3) f32 -> (B,c,n)."""
    _check(points, "points", torch.float32)
    _check(idx, "idx", torch.int32)
    _check(weight, "weight", torch.float32)
    _cuda_only(points, idx, weight)
    B, c, m = points.shape
    n = idx.shape[1]
    out = torch.empty((B, c, n), dtype=torch.float32, device=points.device)
    _lib.call(_lib.pointops(), "sv_three_interpolate_f32", points.device, points.data_ptr(), idx.data_ptr(), weight.data_ptr(),
              B, c, m, n, out.data_ptr())
    return out


def three_interpolate_grad(grad_out, idx, weight, m):
    """interpolate.cpp:71-99.  (B,c,n) -> (B,c,m)."""
    _check(grad_out, "grad_out", torch.float32)
    _check(idx, "idx", torch.int32)
    _check(weight, "weight", torch.float32)
    _cuda_only(grad_out, idx, weight)
    B, c, n = grad_out.shape
    out = torch.empty((B, c, int(m)), dtype=torch.float32, device=grad_out.device)
    _lib.call(_lib.pointops(), "sv_three_interpolate_grad_f32", grad_out.device, grad_out.data_ptr(), idx.data_ptr(),
              weight.data_ptr(), B, c, n, int(m), out.data_ptr())
    return out


def fps_ballquery(xyz, npoint, radius, nsample):
    """Fused extension (not in the reference `_ext`): one pass over xyz (B,N<=1024,3) returning
    (fps_idx (B,npoint) i32, new_xyz (B,npoint,3) f32, ball_idx (B,npoint,nsample) i32), equal to
    furthest_point_sampling + gather_points + ball_query."""
    _check(xyz, "xyz", torch.float32)
    _cuda_only(xyz)
    B, N, _ = xyz.shape
    fps_idx = torch.empty((B, npoint), dtype=torch.int32, device=xyz.device)
    new_xyz = torch.empty((B, npoint, 3), dtype=torch.float32, device=xyz.device)
    ball_idx = torch.empty((B, npoint, nsample), dtype=torch.int32, device=xyz.device)
    if 32 <= N <= 1024:
        _lib.call(_lib.pointops(), "sv_sa_sample_f32", xyz.device, xyz.data_ptr(), B, N, int(npoint), float(radius), int(nsample),
                  fps_idx.data_ptr(), new_xyz.data_ptr(), ball_idx.data_ptr(), 0, 0.0, 0, None, None, None)
    else:
        _lib.call(_lib.pointops(), "sv_fps_ballquery_f32", xyz.device, xyz.data_ptr(), B, N, int(npoint), float(radius),
                  int(nsample), fps_idx.data_ptr(), new_xyz.data_ptr(), ball_idx.data_ptr())
    return fps_idx, new_xyz, ball_idx


def fps_ballquery_scan(xyz, npoint, radius, nsample):
    """The first-generation fused kernel (FPS, then a lane-per-centre scan); kept for N < 32 and as a
    cross-check of sa_sample in the tests."""
    _check(xyz, "xyz", torch.float32)
    _cuda_only(xyz)
    B, N, _ = xyz.shape
    fps_idx = torch.empty((B, npoint), dtype=torch.int32, device=xyz.device)
    new_xyz = torch.empty((B, npoint, 3), dtype=torch.float32, device=xyz.device)
    ball_idx = torch.empty((B, npoint, nsample), dtype=torch.int32, device=xyz.device)
    _lib.call(_lib.pointops(), "sv_fps_ballquery_f32", xyz.device, xyz.data_ptr(), B, N, int(npoint), float(radius), int(nsample),
              fps_idx.data_ptr(), new_xyz.data_ptr(), ball_idx.data_ptr())
    return fps_idx, new_xyz, ball_idx


def sa_sample2(xyz, npoint, radius, nsample, npoint2, radius2, nsample2):
    """Two set-abstraction levels of sampling in one launch (sv_sa_sample_f32); npoint must be 32.
    Returns (fps_idx, new_xyz, ball_idx, fps_idx2, new_xyz2, ball_idx2)."""
    _check(xyz, "xyz", torch.float32)
    _cuda_only(xyz)
    B, N, _ = xyz.shape
    dev = xyz.device
    fps_idx = torch.empty((B, npoint), dtype=torch.int32, device=dev)
    new_xyz = torch.empty((B, npoint, 3), dtype=torch.float32, device=dev)
    ball_idx = torch.empty((B, npoint, nsample), dtype=torch.int32, device=dev)
    fps_idx2 = torch.empty((B, npoint2), dtype=torch.int32, device=dev)
    new_xyz2 = torch.empty((B, npoint2, 3), dtype=torch.float32, device=dev)
    ball_idx2 = torch.empty((B, npoint2, nsample2), dtype=torch.int32, device=dev)
    _lib.call(_lib.pointops(), "sv_sa_sample_f32", xyz.device, xyz.data_ptr(), B, N, int(npoint), float(radius), int(nsample),
              fps_idx.data_ptr(), new_xyz.data_ptr(), ball_idx.data_ptr(), int(npoint2), float(radius2), int(nsample2),
              fps_idx2.data_ptr(), new_xyz2.data_ptr(), ball_idx2.data_ptr())
    return fps_idx, new_xyz, ball_idx, fps_idx2, new_xyz2, ball_idx2
