"""Train-mode PointNet++ set abstraction on the native kernels (config C2, `ObjCls` pre-training with a trainable backbone;
reference: pointnet2_modules.py:34-75, pointnet2_utils.py:291-419, pytorch_utils.py:11-36,67-120).

Channels-LAST formulation: the grouped tensor is a bf16 row matrix X[(b, centre, sample)][channel]; each SharedMLP layer
(Conv2d 1x1 without bias -> BatchNorm2d with BATCH statistics -> ReLU) is one native GEMM (csrc/gemm.cu, forward / dgrad / wgrad)
plus the column-statistic kernels of csrc/pn_train.cu; the neighbourhood max is a max over `nsample` consecutive rows.  The
parameters are the reference's own (`conv.weight (Cout,Cin,1,1)`, `bn.bn.{weight,bias,running_mean,running_var}`): checkpoints and
state_dicts are untouched, running statistics are updated exactly like nn.BatchNorm2d (momentum, unbiased variance)."""
import torch
import torch.nn.functional as F

from . import _lib, native


def _round8(n):
    return (n + 7) // 8 * 8


class _GroupRowsFn(torch.autograd.Function):
    """(xyz (B,N,3) f32, centre (B,np,3) f32 | None, feat (B,N,C) f32 | bf16 | None, idx (B,np,ns) i32 | None) -> X (B*np*ns, Cp) bf16."""

    @staticmethod
    def forward(ctx, xyz, centre, feat, idx, np_, ns):
        B, N, _ = xyz.shape
        C = 0 if feat is None else feat.shape[-1]
        Cp = _round8(3 + C)
        X = torch.empty((B * np_ * ns, Cp), dtype=torch.bfloat16, device=xyz.device)
        xyz, feat = xyz.contiguous(), (feat.contiguous() if feat is not None else None)
        centre = centre.contiguous() if centre is not None else None
        _lib.call(_lib.gps(), "sv_pn_group_rows", xyz.device, xyz.data_ptr(), _lib.ptr(centre), _lib.ptr(feat),
                  1 if (feat is not None and feat.dtype == torch.bfloat16) else 0, _lib.ptr(idx), B, N, C, np_, ns, Cp,
                  X.data_ptr())
        ctx.save_for_backward(idx)
        ctx.meta = (B, N, C, np_, ns, Cp, None if feat is None else feat.dtype)
        return X

    @staticmethod
    def backward(ctx, dX):
        (idx,) = ctx.saved_tensors
        B, N, C, np_, ns, Cp, fdt = ctx.meta
        if C == 0 or not ctx.needs_input_grad[2]:
            return None, None, None, None, None, None
        dX = dX.contiguous()
        dfeat = torch.empty((B, N, C), dtype=torch.float32, device=dX.device)
        _lib.call(_lib.gps(), "sv_pn_group_rows_grad", dX.device, dX.data_ptr(), _lib.ptr(idx), B, N, C, np_, ns, Cp,
                  dfeat.data_ptr())
        return None, None, dfeat.to(fdt), None, None, None


class StatExchange:
    """The column-sum exchange of the SyncBatchNorm layers (csrc/pn_train.cu sv_pn_bn_sync_*; reference: model/objcls.py:33-34
    convert_sync_batchnorm): one symmetric buffer per (device, process group) on top of torch's symmetric-memory allocator, sized
    for C <= CAP and shared by every BatchNorm layer of the backbone — the layers run one after another on one stream, and the
    kernels double-buffer by the parity of the device-resident epoch (each push / finish pair is one exchange)."""
    CAP = 768

    def __init__(self, device, group=None, local=False):
        """local=True: world 1 on an ordinary device buffer, no process group — the same kernels, flags and parity logic."""
        lib = _lib.gps()
        if local:
            self.group, world, rank = None, 1, 0
            self.buf = torch.zeros(lib.sv_pn_sync_floats(self.CAP, 1), dtype=torch.float32, device=device)
            ptrs = [self.buf.data_ptr()]
        else:
            import torch.distributed as dist
            import torch.distributed._symmetric_memory as symm_mem
            self.group = group or dist.group.WORLD
            world, rank = dist.get_world_size(self.group), dist.get_rank(self.group)
            self.buf = symm_mem.empty(lib.sv_pn_sync_floats(self.CAP, world), dtype=torch.float32, device=device)
            self.buf.zero_()
            self.hdl = symm_mem.rendezvous(self.buf, self.group.group_name)
            ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        self._setup(ptrs, world, rank, device)
        torch.cuda.synchronize(device)
        if not local:
            import torch.distributed as dist
            dist.barrier(self.group)      # every rank's buffer (flags included) is zeroed before the first push

    def _setup(self, ptrs, world, rank, device):
        self.world, self.rank = world, rank
        self.peer_bufs = torch.tensor(ptrs, dtype=torch.int64, device=device)
        self.done = torch.zeros(1, dtype=torch.int32, device=device)
        self.epoch_dev = torch.zeros(1, dtype=torch.int32, device=device)   # exchanges completed by this rank (graph-replay safe)

    @classmethod
    def emulated(cls, k, device):
        """Tests only: k ranks on ONE device, each with its own buffer, epoch and done counter, sharing one peer table.  Run
        every rank's push before any rank's finish (one stream): then every flag is already set and no kernel waits."""
        lib = _lib.gps()
        bufs = [torch.zeros(lib.sv_pn_sync_floats(cls.CAP, k), dtype=torch.float32, device=device) for _ in range(k)]
        out = []
        for r in range(k):
            ex = cls.__new__(cls)
            ex.group, ex.buf, ex._all = None, bufs[r], bufs
            ex._setup([b.data_ptr() for b in bufs], k, r, device)
            out.append(ex)
        return out

    def push(self, mode, y, dout=None, stats=None, g32=None, b32=None):
        """mode 0: this rank's column sums of y; mode 1: of g' and g' * xhat (stats = the global mean, rstd)."""
        R, C = y.shape
        assert C <= self.CAP
        lib = _lib.gps()
        scratch = torch.empty(lib.sv_pn_scratch_floats(C), dtype=torch.float32, device=y.device)
        mean, rstd = (stats[0], stats[1]) if stats is not None else (None, None)
        _lib.call(lib, "sv_pn_bn_sync_push", y.device, mode, y.data_ptr(), _lib.ptr(dout), R, C, _lib.ptr(g32), _lib.ptr(b32),
                  _lib.ptr(mean), _lib.ptr(rstd), scratch.data_ptr(), self.peer_bufs.data_ptr(), self.CAP, self.done.data_ptr(),
                  self.world, self.rank, self.epoch_dev.data_ptr())

    def finish_fwd(self, y, g32, b32, eps):
        """-> (relu(BN(y)) bf16, stats (3, C) f32: global mean, rstd, unbiased variance)."""
        R, C = y.shape
        stats = torch.empty((3, C), dtype=torch.float32, device=y.device)
        out = torch.empty_like(y)
        _lib.call(_lib.gps(), "sv_pn_bn_sync_finish_fwd", y.device, y.data_ptr(), R, C, g32.data_ptr(), b32.data_ptr(),
                  float(eps), stats[0].data_ptr(), stats[1].data_ptr(), stats[2].data_ptr(), out.data_ptr(),
                  self.peer_bufs.data_ptr(), self.CAP, self.world, self.rank, self.epoch_dev.data_ptr())
        return out, stats

    def finish_bwd(self, y, dout, stats, g32, b32):
        """-> (dy bf16, dgb (2, C) f32: this rank's d gamma, d beta)."""
        R, C = y.shape
        dy = torch.empty_like(y)
        dgb = torch.empty((2, C), dtype=torch.float32, device=y.device)
        gsum = torch.empty(2 * C + 1, dtype=torch.float32, device=y.device)
        _lib.call(_lib.gps(), "sv_pn_bn_sync_finish_bwd", y.device, y.data_ptr(), dout.data_ptr(), R, C, g32.data_ptr(),
                  b32.data_ptr(), stats[0].data_ptr(), stats[1].data_ptr(), dy.data_ptr(), dgb[0].data_ptr(), dgb[1].data_ptr(),
                  0, gsum.data_ptr(), self.peer_bufs.data_ptr(), self.CAP, self.world, self.rank, self.epoch_dev.data_ptr())
        return dy, dgb


class _ConvBNReLUFn(torch.autograd.Function):
    """out = relu(BatchNorm_batchstats(X W^T)): X (R,Kp) bf16 (zero-padded columns), W = conv.weight (Cout,Cin,1,1) f32.
    ex: a StatExchange for SyncBatchNorm statistics over its ranks (push, then finish, in each direction), or None."""

    @staticmethod
    def conv_fwd(X, weight):
        Cout, Cin = weight.shape[0], weight.shape[1]
        Kp = X.shape[1]
        wb = weight.detach().reshape(Cout, Cin).to(torch.bfloat16)
        if Kp != Cin:
            wb = F.pad(wb, (0, Kp - Cin))
        wb = wb.contiguous()
        return wb, native.linear_fwd(X, wb)

    @staticmethod
    def conv_bwd(X, wb, dy, cin, need_dx=True):
        dX = native.linear_dgrad(dy, wb) if need_dx else None
        dw, _ = native.linear_wgrad(dy, X)
        return dX, dw[:, :cin].reshape(dy.shape[1], cin, 1, 1)

    @staticmethod
    def forward(ctx, X, weight, gamma, beta, eps, ex=None):
        Cout, Cin = weight.shape[0], weight.shape[1]
        R = X.shape[0]
        wb, y = _ConvBNReLUFn.conv_fwd(X, weight)
        g32, b32 = gamma.detach().float().contiguous(), beta.detach().float().contiguous()
        if ex is not None:
            ex.push(0, y)
            out, stats = ex.finish_fwd(y, g32, b32, eps)
        else:
            stats = torch.empty((3, Cout), dtype=torch.float32, device=X.device)     # mean, rstd, unbiased variance
            out = torch.empty_like(y)
            lib = _lib.gps()
            scratch = torch.empty(lib.sv_pn_scratch_floats(Cout), dtype=torch.float32, device=X.device)
            _lib.call(lib, "sv_pn_bn_relu_fwd", X.device, y.data_ptr(), R, Cout, g32.data_ptr(), b32.data_ptr(), float(eps),
                      stats[0].data_ptr(), stats[1].data_ptr(), stats[2].data_ptr(), out.data_ptr(), scratch.data_ptr())
        ctx.save_for_backward(X, wb, y, stats, g32, b32)
        ctx.cin, ctx.ex = Cin, ex
        ctx.mark_non_differentiable(stats)
        return out, stats

    @staticmethod
    def backward(ctx, dout, _dstats):
        X, wb, y, stats, g32, b32 = ctx.saved_tensors
        R, Cout = y.shape
        dout = dout.contiguous()
        if ctx.ex is not None:
            ctx.ex.push(1, y, dout, stats, g32, b32)
            dy, dgb = ctx.ex.finish_bwd(y, dout, stats, g32, b32)
        else:
            dy = torch.empty_like(y)
            dgb = torch.empty((2, Cout), dtype=torch.float32, device=y.device)
            lib = _lib.gps()
            scratch = torch.empty(lib.sv_pn_scratch_floats(Cout), dtype=torch.float32, device=y.device)
            _lib.call(lib, "sv_pn_bn_relu_bwd", y.device, y.data_ptr(), dout.data_ptr(), R, Cout, g32.data_ptr(), b32.data_ptr(),
                      stats[0].data_ptr(), stats[1].data_ptr(), dy.data_ptr(), dgb[0].data_ptr(), dgb[1].data_ptr(), 0,
                      scratch.data_ptr())
        dX, dw = _ConvBNReLUFn.conv_bwd(X, wb, dy, ctx.cin, ctx.needs_input_grad[0])
        return dX, dw, dgb[0], dgb[1], None, None


class _RowGroupMaxFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ns):
        R, C = x.shape
        G = R // ns
        out = torch.empty((G, C), dtype=torch.bfloat16, device=x.device)
        arg = torch.empty((G, C), dtype=torch.uint8, device=x.device)
        _lib.call(_lib.gps(), "sv_pn_rowgroup_max", x.device, x.data_ptr(), G, ns, C, out.data_ptr(), arg.data_ptr())
        ctx.save_for_backward(arg)
        ctx.ns = ns
        return out

    @staticmethod
    def backward(ctx, g):
        (arg,) = ctx.saved_tensors
        G, C = arg.shape
        g = g.contiguous().to(torch.bfloat16)
        gx = torch.empty((G * ctx.ns, C), dtype=torch.bfloat16, device=g.device)
        _lib.call(_lib.gps(), "sv_pn_rowgroup_max_grad", g.device, g.data_ptr(), arg.data_ptr(), G, ctx.ns, C, gx.data_ptr())
        return gx, None


def _update_running_stats(bn, stats):
    """nn.BatchNorm2d's training-mode bookkeeping (momentum update with the UNBIASED batch variance)."""
    if bn.track_running_stats and bn.running_mean is not None:
        with torch.no_grad():
            bn.num_batches_tracked += 1
            m = bn.momentum if bn.momentum is not None else 1.0 / float(bn.num_batches_tracked)
            bn.running_mean.mul_(1 - m).add_(stats[0].to(bn.running_mean.dtype), alpha=m)
            bn.running_var.mul_(1 - m).add_(stats[2].to(bn.running_var.dtype), alpha=m)


_exchanges = {}


def exchange_for(net, device):
    """The StatExchange the net's train-mode BatchNorm layers need on `device`: None when their statistics are local (plain
    BatchNorm2d, or SyncBatchNorm without an initialised process group or over one rank — torch's SyncBatchNorm normalises with
    local statistics then too); False when the layers name different process groups or symmetric memory cannot be set up."""
    syncs = [m for m in net.modules() if isinstance(m, torch.nn.SyncBatchNorm)]
    if not syncs:
        return None
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return None
    groups = {id(m.process_group or dist.group.WORLD): m.process_group or dist.group.WORLD for m in syncs}
    if len(groups) != 1:
        return False
    (group,) = groups.values()
    if dist.get_world_size(group) == 1:
        return None
    key = (str(torch.device(device)), group.group_name)
    if key not in _exchanges:
        try:
            _exchanges[key] = StatExchange(device, group)
        except Exception as e:  # no P2P / unsupported allocator: the generic path with torch's SyncBatchNorm is used instead
            _exchanges[key] = False
            if dist.get_rank() == 0:
                print(f"[sceneverse_b200] native SyncBatchNorm exchange unavailable ({type(e).__name__}: {e}); "
                      "using the generic PointNet++ path")
    return _exchanges[key]


def available(pc, net):
    """Train-mode BatchNorm (or a backbone that needs gradients) on CUDA under bf16 autocast; SyncBatchNorm layers need their
    exchange (exchange_for)."""
    if not (pc.is_cuda and pc.dtype == torch.float32 and torch.is_autocast_enabled("cuda")
            and torch.get_autocast_dtype("cuda") == torch.bfloat16):
        return False
    bns = [m for m in net.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)]
    if not all(type(m) in (torch.nn.BatchNorm2d, torch.nn.SyncBatchNorm) and m.training and m.affine for m in bns):
        return False
    return exchange_for(net, pc.device) is not False


def sample_levels(net, xyz):
    """(new_xyz, ball_idx) of each level of `net` sampled up front, or None for a level sa_forward samples itself.  A net whose
    first two levels are sampled with 32 centres at the first (the GPS encoder) on 32..1024 points gets both levels from ONE
    sa_sample launch (_ext.sa_sample2), whose indices are bit-exact with FPS + gather + ball query (DESIGN.md §1 a1-a3)."""
    from .pointnet2 import _ext
    enc = net.encoder
    if len(enc) >= 2 and enc[0].npoint == 32 and enc[1].npoint is not None and 32 <= xyz.shape[1] <= 1024:
        _, nx1, bi1, _, nx2, bi2 = _ext.sa_sample2(xyz, enc[0].npoint, enc[0].radius, enc[0].nsample,
                                                   enc[1].npoint, enc[1].radius, enc[1].nsample)
        return [(nx1, bi1), (nx2, bi2)] + [None] * (len(enc) - 2)
    return [None] * len(enc)


def sa_forward(sa, xyz, feat, ex=None, sampled=None):
    """One PointnetSAModule in training mode: xyz (B,N,3) f32, feat (B,N,C) point-major (f32 | bf16) -> (new_xyz, (B,np,Cout) bf16).
    ex: the StatExchange of SyncBatchNorm layers, or None.  sampled: this level's (new_xyz, ball_idx) from sample_levels, or None."""
    from .pointnet2 import _ext
    B, N, _ = xyz.shape
    if sampled is not None:
        new_xyz, bidx = sampled
        np_, ns = sa.npoint, sa.nsample
        X = _GroupRowsFn.apply(xyz, new_xyz, feat, bidx, np_, ns)
    elif sa.npoint is not None:
        idx = _ext.furthest_point_sampling(xyz, sa.npoint)
        new_xyz = torch.gather(xyz, 1, idx.long()[..., None].expand(-1, -1, 3)).contiguous()
        bidx = _ext.ball_query(new_xyz, xyz, sa.radius, sa.nsample)
        np_, ns = sa.npoint, sa.nsample
        X = _GroupRowsFn.apply(xyz, new_xyz, feat, bidx, np_, ns)
    else:                                       # GroupAll: one group of all N points, xyz NOT centred (pointnet2_utils.py:389-419)
        new_xyz, np_, ns = None, 1, N
        X = _GroupRowsFn.apply(xyz, None, feat, None, 1, N)
    mlp = sa.mlps[0]
    for j in range(len(sa.mlp_spec) - 1):
        layer = getattr(mlp, f"layer{j}")
        bn = layer.bn.bn
        X, stats = _ConvBNReLUFn.apply(X, layer.conv.weight, bn.weight, bn.bias, bn.eps, ex)
        _update_running_stats(bn, stats)
    out = _RowGroupMaxFn.apply(X, ns)           # (B*np, Cout)
    return new_xyz, out.view(B, np_, -1)


def forward(net, pc, exchange=None):
    """PointNetPP.forward for a trainable backbone: (n, P, 3 + C) f32 -> (n, D).  exchange: the StatExchange of the
    SyncBatchNorm layers; by default exchange_for(net, pc.device)."""
    from . import ops
    ex = exchange if exchange is not None else exchange_for(net, pc.device)
    if ex is False:
        raise RuntimeError("the SyncBatchNorm statistics exchange is unavailable; pn_train.available() routes such a net to "
                           "PointNetPP.forward_generic")
    xyz = pc[..., 0:3].contiguous()
    feat = pc[..., 3:].contiguous() if pc.size(-1) > 3 else None
    for sa, sampled in zip(net.encoder, sample_levels(net, xyz)):
        new_xyz, feat = sa_forward(sa, xyz, feat, ex, sampled)
        xyz = new_xyz if new_xyz is not None else xyz
    return ops.linear(feat.reshape(feat.shape[0], -1), net.fc.weight, net.fc.bias)
