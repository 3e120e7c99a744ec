"""python -m torch.distributed.run --nproc-per-node 2 scripts/objcls_syncbn_2rank.py : native SyncBatchNorm of the trainable
PointNet++ at 2 ranks x 32 objects against one process x 64 objects (native path) and against torch SyncBatchNorm on the generic
fp32 path, then 5 graph-mode ObjClsStep steps.  Rank 0 prints OBJCLS_SYNCBN_OK=True only if every check holds."""
import copy
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.nn.functional as F  # noqa: E402

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dev = torch.device("cuda", lr)
dist.init_process_group("nccl", device_id=dev)
from sceneverse_b200 import pn_train, synthetic, train, weights  # noqa: E402
from sceneverse_b200.modules.pointnet import GPS_SPEC, PointNetPP  # noqa: E402

ok = True


def check(cond, what):
    global ok
    ok = ok and bool(cond)
    if rank == 0 and not cond:
        print("FAILED:", what)


def grads_rule(a, b, tag):
    """test_trainable_backbone_native_path_matches_the_generic_operator_sequence's rule: behind the last neighbourhood max
    tight, the earlier layers by direction."""
    worst = {}
    for (n, p), (_, q) in zip(a.named_parameters(), b.named_parameters()):
        e = (p.grad.float() - q.grad.float()).abs().max().item() / (q.grad.float().abs().max().item() + 1e-8)
        worst[n] = (e, F.cosine_similarity(p.grad.float().flatten(), q.grad.float().flatten(), dim=0).item())
    for n in ("fc.weight", "fc.bias", "encoder.2.mlps.0.layer2.bn.bn.weight", "encoder.2.mlps.0.layer2.bn.bn.bias"):
        check(worst[n][1] > 0.999 and worst[n][0] < 0.1, (tag, n, worst[n]))
    for n, (e, cos) in worst.items():
        check(cos > 0.8, (tag, n, e, cos))
    if rank == 0:
        print(tag, "worst rel", round(max(e for e, _ in worst.values()), 4), "min cos", round(min(c for _, c in worst.values()), 5))


def sum_grads(net):
    for p in net.parameters():
        dist.all_reduce(p.grad, op=dist.ReduceOp.SUM)


torch.manual_seed(0)
base = PointNetPP(**GPS_SPEC)
base.load_state_dict(weights.synthetic_state_dict(base, 0))
base = base.to(dev).train()
full = copy.deepcopy(base)
sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(base))
ref = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(base))
x = torch.from_numpy(synthetic.object_batch(3, 64, 1024, pad_fraction=0.0)).to(dev)
go = torch.randn(64, 768, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
sl = slice(32 * rank, 32 * (rank + 1))
with torch.autocast("cuda", dtype=torch.bfloat16):
    check(pn_train.available(x[sl], sync), "native path refused the SyncBatchNorm net")
    ex = pn_train.exchange_for(sync, dev)
    check(ex is not None and ex is not False and ex.world == 2, "no 2-rank exchange")
    ys = sync(x[sl])
    yf = full(x)                                        # one process, all 64 objects, plain BatchNorm2d
ys.float().backward(go[sl])
yf.float().backward(go)
yr = ref.forward_generic(x[sl])                         # torch SyncBatchNorm, fp32 operator sequence
yr.backward(go[sl])
torch.cuda.synchronize()
e_full = (ys.float() - yf[sl].float()).abs().max().item() / yf.float().abs().max().item()
e_ref = (ys.float() - yr).abs().max().item() / yr.abs().max().item()
check(e_full < 4e-2 and e_ref < 4e-2, ("output", e_full, e_ref))
if rank == 0:
    print("output rel err vs 1x64 native", round(e_full, 5), "vs torch SyncBatchNorm", round(e_ref, 5))
# running statistics: bitwise across ranks (identical global statistics), close to the full-batch and torch values
for (n, b1), (_, b2), (_, b3) in zip(sync.named_buffers(), full.named_buffers(), ref.named_buffers()):
    other = [torch.empty_like(b1) for _ in range(world)]
    dist.all_gather(other, b1)
    check(all(torch.equal(o, b1) for o in other), ("buffer differs across ranks", n))
    if "running" in n:
        for b, tag in ((b2, "1x64"), (b3, "torch")):
            check((b1 - b).abs().max().item() <= 3e-2 * (b.abs().max().item() + 1e-3), (n, tag))
# parameter gradients: this rank's sums (SyncBatchNorm semantics); their sum over ranks is the full-batch gradient
sum_grads(sync)
sum_grads(ref)
grads_rule(sync, full, "grads vs 1x64 native")
grads_rule(sync, ref, "grads vs torch SyncBatchNorm")

# 5 graph-mode ObjClsStep steps: 2 ranks x 32 objects vs one process x 64 objects (dropout off: its masks are per rank)
tf = weights.synthetic_tensor("text_features", (607, 768)).to(dev)
d = [synthetic.scene_batch(7 + i, B=1, O=64, P=1024, all_valid=True) for i in range(5)]
batches = [{k: torch.from_numpy(b[k]).to(dev) for k in ("obj_fts", "obj_labels", "obj_masks")} for b in d]
dp = train.ObjClsStep(dev, tf, dtype=torch.bfloat16, seed=3, cuda_graph=True, num_gpu=2)
one = train.ObjClsStep(dev, tf, dtype=torch.bfloat16, seed=3, cuda_graph=True, num_gpu=1)
check(dp.flat_grads is not None and dp.graph_mode, "ObjClsStep did not take the graph | all-reduce | graph path")
dp.model.dropout.p = one.model.dropout.p = 0.0
l_dp, l_one = [], []
for b in batches:
    half = {k: v[:, sl].contiguous() for k, v in b.items()}
    ld = dp.step(half).clone()
    dist.all_reduce(ld, op=dist.ReduceOp.AVG)
    l_dp.append(float(ld))
    l_one.append(float(one.step(dict(b))))
torch.cuda.synchronize()
for n, t in list(dp.model.named_parameters()) + list(dp.model.named_buffers()):
    other = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(other, t.detach().contiguous())
    check(all(torch.equal(o, t) for o in other), ("ObjClsStep state differs across ranks", n))
# the first call of a graph-mode step runs 3 eager set-up steps + capture on its batch (train.ObjClsStep), so both runs see the
# same sequence of updates; the trajectories agree to the bf16 level of the forward
dev_rel = max(abs(a - b) / abs(b) for a, b in zip(l_dp, l_one))
check(dev_rel < 2e-2, ("loss trajectory", l_dp, l_one))
flag = torch.tensor([int(ok)], device=dev)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)                # a failed check on any rank fails the run
ok = bool(flag.item())
if rank == 0:
    print("loss 2x32", [round(v, 5) for v in l_dp], "1x64", [round(v, 5) for v in l_one])
    print(f"OBJCLS_SYNCBN_OK={ok}")
dist.barrier()
dist.destroy_process_group()
