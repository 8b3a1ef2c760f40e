"""N>1 path on CPU: world_size-2 gloo processes run the sharding / gathering host logic around
a stand-in evaluator (the oracle) and must reproduce the unsharded result exactly."""
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import load_fixture, load_golden_weights


def _init(rank, world, init_file):
    # rendezvous through a file store in the test's temporary directory: unlike a free port picked in advance, no other process can take it
    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method=f"file://{init_file}", rank=rank, world_size=world)


def _worker(rank, world, init_file, q):
    _init(rank, world, init_file)
    try:
        from nabladft_b200.parallel import energy_forces_sharded, max_over_ranks
        from oracle.painn_oc import PaiNNOC

        net = load_golden_weights(PaiNNOC(num_layers=2).double(), torch.float64).eval()
        z, pos, batch = load_fixture([0, 1, 2, 3, 4])
        counts = torch.bincount(batch)
        mol_ptr = torch.zeros(6, dtype=torch.long)
        mol_ptr[1:] = torch.cumsum(counts, 0)

        def fn(z_r, pos_r, ptr_r):
            # one molecule per oracle call: the float64 GEMMs then have the same shapes whichever shard holds the molecule (BLAS may
            # round a row differently when the row count changes), so the results below are comparable bit for bit
            es, fs = [], []
            for a, b in zip(ptr_r[:-1].tolist(), ptr_r[1:].tolist()):
                e, f = net(z_r[a:b], pos_r[a:b].clone(), torch.zeros(b - a, dtype=torch.long))
                es.append(e.detach())
                fs.append(f.detach())
            return torch.cat(es), torch.cat(fs)

        e, f = energy_forces_sharded(fn, z, pos, mol_ptr)
        t = max_over_ranks(10.0 + rank, torch.device("cpu"))
        if rank == 0:
            e_ref, f_ref = fn(z, pos, mol_ptr)
            q.put((torch.equal(e, e_ref), float((f - f_ref).abs().max()), t))
    finally:
        dist.destroy_process_group()


def test_balanced_ranges_cover_everything_once():
    from nabladft_b200.parallel import balanced_ranges

    g = torch.Generator().manual_seed(0)
    for world in (1, 2, 3, 8):
        w = torch.randint(10, 60, (37,), generator=g)
        r = balanced_ranges(w, world)
        assert r[0][0] == 0 and r[-1][1] == 37 and all(a[1] == b[0] for a, b in zip(r, r[1:]))
        loads = [int(w[a:b].sum()) for a, b in r]
        assert max(loads) - min(loads) <= 2 * int(w.max())
    assert balanced_ranges(torch.ones(2), 4)[-1][1] == 2  # more ranks than molecules: empty shards allowed


@pytest.mark.timeout(300)
def test_sharded_energy_forces_world2_gloo(tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    init_file = str(tmp_path / "store")
    procs = [ctx.Process(target=_worker, args=(r, 2, init_file, q)) for r in range(2)]
    for p in procs:
        p.start()
    same_e, df, t = q.get(timeout=240)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    assert same_e and df == 0.0  # per-molecule results do not depend on which rank computed them
    assert t == 11.0  # MAX over ranks


def _grad_worker(rank, world, init_file, q):
    _init(rank, world, init_file)
    try:
        from nabladft_b200.parallel import GradBucket, allreduce_gradients, shard_batch
        from oracle.painn_oc import PaiNNOC

        net = load_golden_weights(PaiNNOC(num_layers=1).double(), torch.float64)
        z, pos, batch = load_fixture([0, 1, 2, 3])
        mol_ptr = torch.zeros(5, dtype=torch.long)
        mol_ptr[1:] = torch.cumsum(torch.bincount(batch), 0)
        target = torch.tensor([-3.0, -2.0, -4.0, -1.0], dtype=torch.float64)

        def loss_sum(z_r, pos_r, ptr_r, t_r):  # SUM over molecules: shards add up to the full-batch loss
            b = torch.repeat_interleave(torch.arange(ptr_r.numel() - 1), ptr_r[1:] - ptr_r[:-1])
            e, _ = net(z_r, pos_r.clone(), b, create_graph=True)
            return ((e - t_r) ** 2).sum()

        z_r, pos_r, ptr_r, (m0, m1) = shard_batch(z, pos, mol_ptr, rank, world)
        net.zero_grad()
        if m1 > m0:
            loss_sum(z_r, pos_r, ptr_r, target[m0:m1]).backward()
        n = allreduce_gradients(net.parameters(), average=False)
        got = [p.grad.clone() for p in net.parameters()]
        # the pre-flattened bucket (what bench.py's training sub-record uses): gradients accumulate into views of ONE buffer
        bucket = GradBucket(net.parameters())
        bucket.zero()
        if m1 > m0:
            loss_sum(z_r, pos_r, ptr_r, target[m0:m1]).backward()
        views_alive = all(p.grad.data_ptr() >= bucket.flat.data_ptr() and p.grad.data_ptr() < bucket.flat.data_ptr() + bucket.flat.numel() * 8
                          for p in net.parameters())
        n2 = bucket.allreduce(average=False)
        got2 = [p.grad.clone() for p in net.parameters()]
        if rank == 0:
            net.zero_grad()
            loss_sum(z, pos, mol_ptr, target).backward()
            err = max(float((g - p.grad).abs().max() / (p.grad.abs().max() + 1e-30)) for g, p in zip(got, net.parameters()))
            err2 = max(float((g - p.grad).abs().max() / (p.grad.abs().max() + 1e-30)) for g, p in zip(got2, net.parameters()))
            q.put((n, max(err, err2) if (views_alive and n2 == n) else 1.0))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_gradient_allreduce_world2_gloo_equals_full_batch_gradient(tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    init_file = str(tmp_path / "store")
    procs = [ctx.Process(target=_grad_worker, args=(r, 2, init_file, q)) for r in range(2)]
    for p in procs:
        p.start()
    n, err = q.get(timeout=240)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    assert n > 100000 and err < 1e-12  # one flat all-reduce reproduces the single-process gradient (float64 oracle model)
