"""normalise + all-gather over NVLink peer memory (csrc/norm_allgather.cu) on top of torch's symmetric-memory
allocator (the rendezvous / peer mapping is torch.distributed plumbing; the exchange itself is one native kernel)."""
import torch
import torch.distributed as dist

from . import _lib

_state = {}


class FusedNormGather:
    SIG_WORDS = 64

    def __init__(self, n, D, device, group=None, local=False):
        """local=True: a single-rank self-exchange on an ordinary device buffer (world = 1, no process group) — the same
        kernel, epoch flags and parity logic, used by the single-GPU parity test."""
        self.n, self.D = n, D
        if local:
            self.group, self.world, self.rank = None, 1, 0
            self.buf = torch.zeros(2 * 2 * n * D + self.SIG_WORDS, dtype=torch.float32, device=device)
            ptrs = [self.buf.data_ptr()]
        else:
            import torch.distributed._symmetric_memory as symm_mem
            self.group = group or dist.group.WORLD
            self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
            self.buf = symm_mem.empty(2 * 2 * self.world * n * D + self.SIG_WORDS, dtype=torch.float32, device=device)
            self.buf.zero_()
            self.hdl = symm_mem.rendezvous(self.buf, self.group.group_name)
            ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        data_floats = 2 * 2 * self.world * n * D
        self.data_floats = data_floats
        self.peer_bufs = torch.tensor(ptrs, dtype=torch.int64, device=device)
        self.peer_sigs = torch.tensor([p + 4 * data_floats for p in ptrs], dtype=torch.int64, device=device)
        self.done = torch.zeros(1, dtype=torch.int32, device=device)
        self.epoch_dev = torch.zeros(1, dtype=torch.int32, device=device)  # the kernel's own epoch word (graph-replay safe)
        torch.cuda.synchronize(device)
        if not local:
            dist.barrier(self.group)  # every rank's buffer (incl. signal words) is zeroed before the first exchange

    def __call__(self, a, b):
        """a, b: (n,D) -> (normalize(a) gathered (world*n,D), normalize(b) gathered) as fresh tensors.
        The kernel writes the parity half selected by ITS device-resident epoch, and the result is copied out of the half
        selected by the SAME device word (an index_select with a device index), so eager calls and CUDA-graph replays
        agree for any number of exchanges per step; copying out also means nothing (autograd included) keeps a view of
        the symmetric buffer, so a faster rank's later exchange can never overwrite data that is still to be read."""
        a = a.detach().float().contiguous()
        b = b.detach().float().contiguous()
        assert a.shape == (self.n, self.D) and b.shape == (self.n, self.D)
        _lib.call(_lib.gps(), "sv_normalize_allgather_dev_f32", a.device, a.data_ptr(), b.data_ptr(), self.n, self.D,
                  self.peer_bufs.data_ptr(), self.peer_sigs.data_ptr(), self.done.data_ptr(), self.world, self.rank,
                  self.epoch_dev.data_ptr())
        wn = self.world * self.n
        parity = (self.epoch_dev & 1).long()          # the kernel stored the epoch it used; stream-ordered after it
        out = self.buf[:self.data_floats].view(2, 2, wn, self.D).index_select(0, parity)[0]
        return out[0], out[1]


def get(n, D, device):
    """One exchange object per (n, D, device); None if symmetric memory cannot be set up on this system."""
    key = (n, D, str(device))
    if key not in _state:
        try:
            _state[key] = FusedNormGather(n, D, device)
        except Exception as e:  # no P2P / unsupported allocator: the NCCL path of losses.all_gather is used instead
            _state[key] = None
            if dist.get_rank() == 0:
                print(f"[sceneverse_b200] fused normalise+all-gather unavailable ({type(e).__name__}: {e}); using NCCL all_gather")
    return _state[key]
