"""2-GPU tests (run on a machine with >= 2 H100s): the data-parallel step --
fused peer-memory optimizer ("p2p") and NCCL all-reduce ("nccl") -- equals the single-GPU step on
the concatenated global batch; sharded ranking equals full ranking."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
mode = sys.argv[2]
from ampligraph_b200.engine import KGEEngine
from ampligraph_b200.parallel import DataParallelTrainer, allreduce_sum_, batch_slot, row_shard, tables_close
local = int(os.environ["LOCAL_RANK"]); torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
rank, world = dist.get_rank(), dist.get_world_size()
rng = np.random.default_rng(0)
model, E, R, k, eta, B, steps = "ComplEx", 3000, 11, 64, 6, 512, 4
K = 2 * k
ent = rng.uniform(-.2, .2, (E, K)).astype(np.float32); rel = rng.uniform(-.2, .2, (R, K)).astype(np.float32)
data = np.stack([rng.integers(0, E, steps*world*B), rng.integers(0, R, steps*world*B), rng.integers(0, E, steps*world*B)], 1).astype(np.int32)
neg_ent = rng.integers(0, E, (steps*world, B*eta)).astype(np.int32); neg_keep = rng.integers(0, 2, (steps*world, B*eta)).astype(np.uint8)
dev = lambda a: torch.as_tensor(a).cuda().contiguous()
regs = [{"p": 2, "lambda": 1e-3}, {"p": 3, "lambda": 2e-3}]   # a different regulariser per table: the exchange kernel switches at the ent|rel boundary
mk = lambda alloc: KGEEngine(model, k, eta, E, R, loss="self_adversarial", optimizer="adam",
                             optimizer_params={"learning_rate": 1e-2}, regularizer=regs, device=local, table_alloc=alloc)
try:
    dp = DataParallelTrainer(mk, mode=mode)
except RuntimeError as e:
    if mode == "nvls" and "multicast" in str(e):   # no NVLS on this box: nothing to test
        print("rank", int(os.environ["RANK"]), mode, "ok (skipped: %s)" % e); dist.destroy_process_group(); raise SystemExit(0)
    raise
assert dp.mode == mode, (dp.mode, getattr(dp, "p2p_error", None))
dp.eng.set_embeddings(ent, rel)
for i in range(steps):
    j = batch_slot(i, world, rank, steps*world)
    dp.train_step(dev(data[j*B:(j+1)*B]), (dev(neg_ent[j]), dev(neg_keep[j])))
torch.cuda.synchronize()
got_e, got_r = (x.cpu().numpy() for x in dp.eng.get_embeddings())
# single-GPU run on the concatenated global batches (rank 0 only needs to check; all ranks do)
ref = mk(None)
ref.set_embeddings(ent, rel)
for i in range(steps):
    js = [batch_slot(i, world, r, steps*world) for r in range(world)]
    t = np.concatenate([data[j*B:(j+1)*B] for j in js])
    # tile order for the concatenated batch: row jj*Bg + i
    ne = np.concatenate([neg_ent[j].reshape(eta, B) for j in js], axis=1).reshape(-1)
    nk = np.concatenate([neg_keep[j].reshape(eta, B) for j in js], axis=1).reshape(-1)
    ref.train_step(dev(t), (dev(ne), dev(nk)))
ref_e, ref_r = (x.cpu().numpy() for x in ref.get_embeddings())
ok_e, err_e = tables_close(got_e, ref_e, ent, rtol=2e-4); ok_r, err_r = tables_close(got_r, ref_r, rel, rtol=2e-4)
print("rank", rank, mode, "max err / max update: ent %.2e rel %.2e" % (err_e, err_r), flush=True)
assert ok_e and ok_r, (err_e, err_r)
loss = dp.reduce_loss_().sum().item(); ref_loss = ref.read_loss()   # batch loss + regulariser loss, summed over ranks
assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss), (loss, ref_loss)
# the lazy rule is refused with replicated tables (ADVICE r1)
try:
    DataParallelTrainer(lambda alloc: KGEEngine(model, k, eta, E, R, optimizer="lazy_adam", device=local, table_alloc=alloc), mode=mode)
    raise SystemExit("lazy_adam was accepted")
except NotImplementedError:
    pass
# every replica holds the same table
chk = torch.tensor([float(np.abs(got_e).sum())], device="cuda", dtype=torch.float64)
lo = chk.clone(); dist.all_reduce(lo, op=dist.ReduceOp.MIN); hi = chk.clone(); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
assert lo.item() == hi.item()
# sharded ranking: each rank counts against its row shard, counts are summed
q = dev(data[:64])
lo_r, hi_r = row_shard(E, world, rank)
for strategy in ("worst", "middle"):
    cnt = torch.zeros((64, 3), dtype=torch.int32, device="cuda")
    ref.rank(q, "o", strategy, cand_begin=lo_r, n_cand=hi_r - lo_r, counts=cnt)
    allreduce_sum_([cnt])
    assert (ref.finalize_ranks(cnt, strategy) == ref.rank(q, "o", strategy)).all()
dist.destroy_process_group()
print("rank", rank, mode, "ok")
'''


@pytest.mark.parametrize("mode", ["nccl", "p2p", "nvls"])
def test_data_parallel_step_two_gpus(tmp_path, mode):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29621", str(script), ROOT, mode]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=420)
    assert out.returncode == 0, out.stdout[-4000:]
    assert out.stdout.count(mode + " ok") >= 2


_SHARD_WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from ampligraph_b200.engine import KGEEngine
from ampligraph_b200.parallel import ShardedTrainer, batch_slot, tables_close
local = int(os.environ["LOCAL_RANK"]); torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
rank, world = dist.get_rank(), dist.get_world_size()
rng = np.random.default_rng(0)
for model, k, opt in (("RotatE", 24, "adam"), ("ComplEx", 40, "adam"), ("ComplEx", 40, "lazy_adam"), ("DistMult", 300, "lazy_adam")):
    E, R, eta, B, steps = 1001, 7, 5, 300, 3   # E not divisible by world: last shard is short
    if k == 300: eta = 40                      # non-resident geometry: negative groups + the row stash through peer memory
    K = k if model in ("TransE", "DistMult") else 2 * k
    ent = rng.uniform(-.2, .2, (E, K)).astype(np.float32); rel = rng.uniform(-.2, .2, (R, K)).astype(np.float32)
    data = np.stack([rng.integers(0, E, steps*world*B), rng.integers(0, R, steps*world*B), rng.integers(0, E, steps*world*B)], 1).astype(np.int32)
    neg_ent = rng.integers(0, E, (steps*world, B*eta)).astype(np.int32); neg_keep = rng.integers(0, 2, (steps*world, B*eta)).astype(np.uint8)
    dev = lambda a: torch.as_tensor(a).cuda().contiguous()
    kw = dict(loss="self_adversarial", optimizer=opt, optimizer_params={"learning_rate": 1e-3})
    tr = ShardedTrainer(model, k, eta, E, R, local, **kw)
    tr.set_embeddings(ent, rel)
    ref = KGEEngine(model, k, eta, E, R, device=local, **kw)
    ref.set_embeddings(ent, rel)
    for i in range(steps):
        j = batch_slot(i, world, rank, steps*world)
        tr.train_step(dev(data[j*B:(j+1)*B]), (dev(neg_ent[j]), dev(neg_keep[j])), step=i)
        js = [batch_slot(i, world, r, steps*world) for r in range(world)]
        t = np.concatenate([data[jj*B:(jj+1)*B] for jj in js])
        ne = np.concatenate([neg_ent[jj].reshape(eta, B) for jj in js], axis=1).reshape(-1)
        nk = np.concatenate([neg_keep[jj].reshape(eta, B) for jj in js], axis=1).reshape(-1)
        ref.train_step(dev(t), (dev(ne), dev(nk)), step=i)
    got_e, got_r = (x.numpy() for x in tr.get_embeddings())
    ref_e, ref_r = (x.cpu().numpy() for x in ref.get_embeddings())
    ok_e, err_e = tables_close(got_e, ref_e, ent); ok_r, err_r = tables_close(got_r, ref_r, rel)
    print("rank", rank, model, k, opt, "max err / max update: ent %.2e rel %.2e" % (err_e, err_r), flush=True)
    assert ok_e and ok_r, (model, k, opt, err_e, err_r)
    # sharded ranking == ranking on the gathered table (bit-exact)
    ref.set_embeddings(got_e, got_r)
    q = dev(data[:48])
    filt = [sorted(set(rng.integers(0, E, 6).tolist())) for _ in range(48)]
    off = dev(np.concatenate([[0], np.cumsum([len(f) for f in filt])]).astype(np.int64)); idx = dev(np.concatenate(filt).astype(np.int32))
    for side in ("s", "o"):
        for strategy in ("worst", "middle", "best"):
            assert (tr.rank_counts(q, side, strategy, off, idx) == ref.rank(q, side, strategy, off, idx)).all(), (model, side, strategy)
    tr.close(); ref.close()
dist.destroy_process_group()
print("rank", rank, "sharded ok")
'''


def test_row_sharded_tables_two_gpus(tmp_path):
    """Row-sharded entity table over 2 GPUs (gathers/scatters through NVLink peer memory inside the
    fused kernel) == single-GPU training on the concatenated batch; sharded ranking bit-exact."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(_SHARD_WORKER)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29623", str(script), ROOT]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=420)
    assert out.returncode == 0, out.stdout[-4000:]
    assert out.stdout.count("sharded ok") >= 2
