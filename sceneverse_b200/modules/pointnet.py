"""PointNet++ object encoder (reference: modules/layers/pointnet.py:22-63 `PointNetPP`,
modules/third_party/pointnet2/pointnet2_modules.py:34-161 `PointnetSAModule`).

Same constructor, same forward contract ((B,P,3+C) -> (B,D)) and the same state_dict keys
(`encoder.{i}.mlps.0.layer{j}.conv.weight`, `...bn.bn.*`, `fc.*`, SURVEY.md §8b) as the reference.

Two execution paths, both on the GPU, both through the native point-op library:
  * fused (the GPS configuration with BatchNorm in eval mode — the frozen backbone of
    all_pretrain.yaml): sa_sample (FPS + ball query, two levels, one launch) -> wgmma
    set-abstraction MLP kernels (gather + 3 GEMMs + max fused) -> SA3/fc;
  * generic (any other PointnetSAModule stack, or train-mode BatchNorm): the reference's operator
    sequence on the native `_ext` kernels with torch conv/BN (needed for `ObjCls` pre-training).
"""
import torch
import torch.nn.functional as F
from torch import nn

from .. import _lib, native, pointnet2_utils
from ..pointnet2 import _ext


# ------------------------------------------------------------------ parameter containers (key-compatible)
class _BN(nn.Sequential):
    def __init__(self, c):
        super().__init__()
        self.add_module("bn", nn.BatchNorm2d(c))


class _ConvBNReLU(nn.Sequential):
    """pytorch_utils.py:67-120 with bn=True: Conv2d(1x1, bias=False) -> BatchNorm2d -> ReLU."""

    def __init__(self, cin, cout):
        super().__init__()
        conv = nn.Conv2d(cin, cout, kernel_size=(1, 1), bias=False)
        nn.init.kaiming_normal_(conv.weight)
        self.add_module("conv", conv)
        self.add_module("bn", _BN(cout))
        self.add_module("activation", nn.ReLU(inplace=True))


class _SharedMLP(nn.Sequential):
    def __init__(self, spec):
        super().__init__()
        for i in range(len(spec) - 1):
            self.add_module(f"layer{i}", _ConvBNReLU(spec[i], spec[i + 1]))


class _SAModule(nn.Module):
    def __init__(self, npoint, radius, nsample, mlp, use_xyz=True):
        super().__init__()
        self.npoint, self.radius, self.nsample = npoint, radius, nsample
        mlp = list(mlp)
        if use_xyz:
            mlp[0] += 3
        self.mlp_spec = mlp
        self.groupers = nn.ModuleList([
            pointnet2_utils.QueryAndGroup(radius, nsample, use_xyz=use_xyz) if npoint is not None
            else pointnet2_utils.GroupAll(use_xyz)])
        self.mlps = nn.ModuleList([_SharedMLP(mlp)])

    def forward(self, xyz, features):
        """Reference operator sequence (pointnet2_modules.py:34-75) on the native kernels."""
        new_xyz = None
        if self.npoint is not None:
            idx = pointnet2_utils.furthest_point_sample(xyz, self.npoint)
            new_xyz = pointnet2_utils.gather_operation(xyz.transpose(1, 2).contiguous(), idx).transpose(1, 2).contiguous()
        new_features = self.groupers[0](xyz, new_xyz, features)
        new_features = self.mlps[0](new_features)
        new_features = F.max_pool2d(new_features, kernel_size=[1, new_features.size(3)]).squeeze(-1)
        return new_xyz, new_features


# ------------------------------------------------------------------ packing for the wgmma kernels
def fold_bn(conv_w, bn, eps=None):
    """(Cout,Cin,1,1) conv weight + eval-mode BatchNorm2d -> (W' (Cout,Cin) f32 with the scale folded, shift (Cout) f32)."""
    eps = bn.eps if eps is None else eps
    scale = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + eps)
    shift = bn.bias.detach().float() - bn.running_mean.detach().float() * scale
    return conv_w.detach().float().reshape(conv_w.shape[0], -1) * scale[:, None], shift


def to_umma_kmajor(w):
    """(N,K) with K % 8 == 0 -> bf16 bytes in the canonical no-swizzle K-major wgmma layout [K/8][N][8] (sm90.cuh)."""
    n, k = w.shape
    assert k % 8 == 0
    return w.to(torch.bfloat16).reshape(n, k // 8, 8).permute(1, 0, 2).contiguous()


def to_umma_sw128(w):
    """(N,K) -> bf16 operand image for csrc/sa_mlp.cu: the first floor(K/64)*64 columns as SWIZZLE_128B K-major slabs
    ([slab][N][8 chunks][8], chunk position = chunk ^ (n & 7)), the remaining (< 64) columns as a no-swizzle K-major
    tail ([K/8][N][8])."""
    n, k = w.shape
    ksw = (k // 64) * 64
    wb = w.to(torch.bfloat16)
    parts = []
    if ksw:
        sl = wb[:, :ksw].reshape(n, ksw // 64, 8, 8)                      # (n, slab, chunk, 8)
        pos = torch.arange(8, device=w.device)[None, :] ^ (torch.arange(n, device=w.device)[:, None] & 7)  # chunk stored at position p
        sl = torch.gather(sl, 2, pos[:, None, :, None].expand(n, ksw // 64, 8, 8))   # out[n,s,p] = in[n,s,p ^ (n&7)]
        parts.append(sl.permute(1, 0, 2, 3).contiguous().reshape(-1))
    if k > ksw:
        parts.append(to_umma_kmajor(wb[:, ksw:].contiguous()).reshape(-1))
    return torch.cat(parts).contiguous()


def pack_sa_params(level, layers):
    """layers = 3 x (W' (Cout,Cin) f32, shift (Cout) f32) in the REFERENCE channel order
    (cat([grouped_xyz(3), grouped_features(C)]), pointnet2_utils.py:354-356).  Returns a uint8 CUDA tensor laid out as
    sv_sa1_mlp_bf16 / sv_sa2_mlp_bf16 expect."""
    (w1, s1), (w2, s2), (w3, s3) = layers
    dev = w1.device
    if level == 1:
        k1p = 16
        w1p = torch.zeros(w1.shape[0], k1p, device=dev)
        w1p[:, :6] = w1  # [dx dy dz r g b | 0...]
    else:
        k1p = 144
        w1p = torch.zeros(w1.shape[0], k1p, device=dev)
        w1p[:, :128] = w1[:, 3:]   # kernel column order: features first ...
        w1p[:, 128:131] = w1[:, :3]  # ... then xyz - centre
    parts = [to_umma_sw128(w1p).view(torch.uint8).reshape(-1), to_umma_sw128(w2).view(torch.uint8).reshape(-1),
             to_umma_sw128(w3).view(torch.uint8).reshape(-1),
             torch.cat([s1, s2, s3]).float().contiguous().view(torch.uint8).reshape(-1)]
    buf = torch.cat(parts).contiguous()
    want = _lib.gps().sv_sa_mlp_param_bytes(level)
    assert buf.numel() == want, (buf.numel(), want)
    return buf


GPS_SPEC = dict(sa_n_points=[32, 16, None], sa_n_samples=[32, 32, None], sa_radii=[0.2, 0.4, None],
                sa_mlps=[[3, 64, 64, 128], [128, 128, 128, 256], [256, 256, 512, 768]])


class PointNetPP(nn.Module):
    def __init__(self, sa_n_points, sa_n_samples, sa_radii, sa_mlps, bn=True, use_xyz=True):
        super().__init__()
        n_sa = len(sa_n_points)
        if not (n_sa == len(sa_n_samples) == len(sa_radii) == len(sa_mlps)):
            raise ValueError('Lens of given hyper-params are not compatible')
        if not bn:
            raise NotImplementedError("the reference GPS encoder always uses bn=True")
        self.spec = dict(sa_n_points=list(sa_n_points), sa_n_samples=list(sa_n_samples), sa_radii=list(sa_radii),
                         sa_mlps=[list(m) for m in sa_mlps])
        self.encoder = nn.ModuleList([
            _SAModule(sa_n_points[i], sa_radii[i], sa_n_samples[i], sa_mlps[i], use_xyz) for i in range(n_sa)])
        out_n_points = sa_n_points[-1] if sa_n_points[-1] is not None else 1
        self.fc = nn.Linear(out_n_points * sa_mlps[-1][-1], sa_mlps[-1][-1])
        self._packed = None
        self._packed_key = None

    # -------------------------------------------------------------- helpers
    def _bn_all_eval(self):
        return all(not m.training for m in self.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm))

    def fused_available(self, pts):
        return (self.spec == GPS_SPEC and pts.is_cuda and pts.dtype == torch.float32 and pts.size(-1) == 6
                and 32 <= pts.size(1) <= 1024 and self._bn_all_eval() and not self._needs_grad())

    def _needs_grad(self):
        return torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())

    def _pack(self):
        key = tuple((p.data_ptr(), p._version) for p in list(self.parameters()) + list(self.buffers()))
        if self._packed is None or self._packed_key != key:
            packed = []
            for lvl in (0, 1, 2):
                mlp = self.encoder[lvl].mlps[0]
                layers = [fold_bn(getattr(mlp, f"layer{j}").conv.weight, getattr(mlp, f"layer{j}").bn.bn) for j in range(3)]
                packed.append(layers)
            # SA3 (GroupAll): layer-1 input channels [xyz(3) | feat(256)] re-ordered to [feat(256) | xyz(3) | 0-pad(13)] so
            # that the bf16 operand rows are 16-byte aligned for TMA (K = 272)
            (w1, s1), (w2, s2), (w3, s3) = packed[2]
            w1p = torch.zeros(w1.shape[0], 272, device=w1.device)
            w1p[:, :256], w1p[:, 256:259] = w1[:, 3:], w1[:, :3]
            bf = torch.bfloat16
            sa3 = [(w1p.to(bf).contiguous(), s1.float().contiguous()), (w2.to(bf).contiguous(), s2.float().contiguous()),
                   (w3.to(bf).contiguous(), s3.float().contiguous())]
            fc = (self.fc.weight.detach().to(bf).contiguous(), self.fc.bias.detach().float().contiguous())
            self._packed = dict(sa1=pack_sa_params(1, packed[0]), sa2=pack_sa_params(2, packed[1]), sa3=sa3, fc=fc)
            self._packed_key = key
        return self._packed

    @torch.no_grad()
    def refresh_pack_(self):
        """Re-pack the current weights INTO the existing packed images (a captured CUDA graph holds their addresses and the
        host check of _pack never runs during replays).  Nothing to do if the fused path never packed."""
        old = self._packed
        if old is None:
            return
        self._packed = None
        new = self._pack()
        pairs = [(old["sa1"], new["sa1"]), (old["sa2"], new["sa2"])]
        pairs += [(a, b) for (oa, ob), (na, nb) in zip(old["sa3"] + [old["fc"]], new["sa3"] + [new["fc"]])
                  for a, b in ((oa, na), (ob, nb))]
        for dst, src in pairs:
            if dst.shape != src.shape or dst.dtype != src.dtype:
                raise RuntimeError("PointNet++ packed weights cannot be refreshed in place: their layout changed")
            if dst.data_ptr() != src.data_ptr():       # the fp32 fc bias is the parameter itself: already current
                dst.copy_(src)
        self._packed = old          # _pack() left the key of the current weights

    def train(self, mode=True):
        """Leaving train mode re-derives the packed eval-mode images in place from the current weights and BatchNorm
        running statistics.  Training changes them without a host-visible version bump (the flat AdamW of a captured step
        writes through the flat buffer, replayed BatchNorm updates write the buffers), so neither _pack's key nor a
        captured evaluation graph, which holds the images' addresses, would notice; EvalRunner.run and model.eval() both
        pass through here before they read the images."""
        if not mode and self.training and self._packed is not None:
            self.refresh_pack_()
        return super().train(mode)

    # -------------------------------------------------------------- forward
    def forward(self, features):
        """@param features: (B*N_objects, N_points, 3 + C)  ->  (B*N_objects, D)"""
        if self.fused_available(features):
            return self.forward_fused(features)
        from .. import pn_train
        if pn_train.available(features, self):
            # trainable backbone under bf16 autocast (ObjCls pre-training): channels-last native path — wgmma GEMMs for the
            # 1x1 convolutions, batch-statistic BatchNorm / max kernels of csrc/pn_train.cu
            return pn_train.forward(self, features)
        return self.forward_generic(features)

    def forward_generic(self, pc):
        xyz = pc[..., 0:3].contiguous()
        feats = pc[..., 3:].transpose(1, 2).contiguous() if pc.size(-1) > 3 else None
        for sa in self.encoder:
            xyz, feats = sa(xyz, feats)
        return self.fc(feats.view(feats.size(0), -1))

    @torch.no_grad()
    def forward_fused(self, pts, return_intermediates=False):
        pk = self._pack()
        B, P, _ = pts.shape
        pts = pts.contiguous()
        xyz = pts[..., :3].contiguous()
        sa1, sa2 = self.encoder[0], self.encoder[1]
        fi1, nx1, bi1, fi2, nx2, bi2 = _ext.sa_sample2(xyz, sa1.npoint, sa1.radius, sa1.nsample,
                                                       sa2.npoint, sa2.radius, sa2.nsample)
        feat1 = torch.empty((B, 32, 128), dtype=torch.bfloat16, device=pts.device)
        _lib.call(_lib.gps(), "sv_sa1_mlp_bf16", pts.device, pts.data_ptr(), nx1.data_ptr(), bi1.data_ptr(), pk["sa1"].data_ptr(),
                  B, P, sa1.nsample, feat1.data_ptr())
        feat2 = torch.empty((B, 16, 256), dtype=torch.bfloat16, device=pts.device)
        _lib.call(_lib.gps(), "sv_sa2_mlp_bf16", pts.device, nx1.data_ptr(), feat1.data_ptr(), nx2.data_ptr(), bi2.data_ptr(),
                  pk["sa2"].data_ptr(), B, 32, sa2.nsample, feat2.data_ptr())
        # SA3 (GroupAll over the 16 points: 259->256->512->768, BN folded, ReLU, max over the points) + fc, as four
        # wgmma GEMMs with fused shift/ReLU (and row-group max) epilogues.  xyz is NOT centred here (GroupAll,
        # pointnet2_utils.py:389-419).
        x = torch.zeros((B * 16, 272), dtype=torch.bfloat16, device=pts.device)
        x[:, :256] = feat2.view(B * 16, 256)
        x[:, 256:259] = nx2.reshape(B * 16, 3).to(torch.bfloat16)
        (w1, s1), (w2, s2), (w3, s3) = pk["sa3"]
        x = native.gemm(x, w1, s1, "relu")
        x = native.gemm(x, w2, s2, "relu")
        g = native.gemm(x, w3, s3, "relu", rowmax=16)                 # (B,768) bf16: max over the 16 points
        out = native.gemm(g, pk["fc"][0], pk["fc"][1], out_dtype=torch.float32)
        if return_intermediates:
            return out, dict(fps_idx=fi1, new_xyz=nx1, ball_idx=bi1, fps_idx2=fi2, new_xyz2=nx2, ball_idx2=bi2,
                             feat1=feat1, feat2=feat2)
        return out
