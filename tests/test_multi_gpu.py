"""N > 1: the row-shard plumbing on CPU (gloo, world_size 2) and, when two GPUs are visible, the
sharded training step against the single-GPU one."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, n, balanced=False):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from sslrec_b200.parallel import RowShard
    n_user = n // 3
    from sslrec_b200.parallel import balanced_bounds
    # unequal blocks: boundaries that balance a skewed per-row weight (one hub row holds a third of the weight)
    w_u, w_i = torch.ones(n_user), torch.ones(n - n_user)
    w_i[0] = float(n)
    ub, ib = balanced_bounds(w_u, world), balanced_bounds(w_i, world)
    assert ub[0] == 0 and ub[-1] == n_user and ib[-1] == n - n_user and ib[1] <= max(1, (n - n_user) // world)      # the hub's block is short
    sh = RowShard(dist, rank, world, n, n_user=n_user, shard_propagation=True, user_bounds=ub if balanced else None, item_bounds=ib if balanced else None)
    assert sh.transport == 'nccl'            # gloo: collectives after the launch, no peer stores
    # every global row belongs to exactly one rank, and every rank owns rows of both sides
    owned = torch.zeros(n)
    (u0, u1), (i0, i1) = sh.ranges
    owned[u0:u1] += 1
    owned[i0:i1] += 1
    assert u1 <= n_user <= i0 and sh.n_local == (u1 - u0) + (i1 - i0)
    dist.all_reduce(owned)
    assert torch.equal(owned, torch.ones(n))
    # a table whose owned rows were written locally becomes complete on every rank
    full = torch.arange(n * 2 * 3, dtype=torch.float32).view(n, 2, 3)
    tb = sh.table('x', (n, 2, 3), 'cpu')
    assert sh.table('x', (n, 2, 3), 'cpu') is tb and not tb.peer_ptrs
    tb.t.fill_(-1.0)
    tb.t[u0:u1] = full[u0:u1]
    tb.t[i0:i1] = full[i0:i1]
    sh.sync_rows(tb)
    assert torch.equal(tb.t, full)
    # the sharded optimizer's parameter exchange (nccl transport path) completes the table the same way
    from sslrec_b200.optim import FusedAdam
    p_u, p_i = torch.nn.Parameter(torch.full((n_user, 4), -1.0)), torch.nn.Parameter(torch.full((n - n_user, 4), -1.0))
    want_u, want_i = torch.arange(n_user * 4.0).view(n_user, 4), 100 + torch.arange((n - n_user) * 4.0).view(n - n_user, 4)
    p_u.data[u0:u1] = want_u[u0:u1]
    p_i.data[i0 - n_user:i1 - n_user] = want_i[i0 - n_user:i1 - n_user]
    opt = FusedAdam([p_u, p_i], row_shards={id(p_u): (u0, u1, [], sh.user_bounds), id(p_i): (i0 - n_user, i1 - n_user, [], sh.item_bounds)}, comm=sh)
    opt._after_sharded_step([p_u, p_i])
    assert torch.equal(p_u.data, want_u) and torch.equal(p_i.data, want_i)
    # InfoNCE table sharding: side ranges split without gaps
    lo_u, hi_u = sh.side_range(0, n_user)
    lo_i, hi_i = sh.side_range(n_user, n - n_user)
    cnt = torch.tensor([hi_u - lo_u, hi_i - lo_i], dtype=torch.float32)
    dist.all_reduce(cnt)
    assert cnt.tolist() == [n_user, n - n_user]
    # partial (row sum, weighted sum) of a sharded softmax contraction all-reduce to the full one
    g = torch.Generator().manual_seed(0)
    a, t = torch.randn(5, 4, generator=g), torch.randn(n, 4, generator=g)
    lo, hi = sh.side_range(0, n)
    e = torch.exp(a @ t[lo:hi].T)
    red = torch.cat([e @ t[lo:hi], e.sum(1, keepdim=True)], 1)
    blk = torch.zeros(sh.side_block(n), 4)
    blk[:hi - lo] = t[lo:hi]
    assert torch.equal(sh.allgather_side(blk, n), t)
    sh.allreduce_sum(red)
    ef = torch.exp(a @ t.T)
    assert torch.allclose(red[:, :4], ef @ t, rtol=1e-5) and torch.allclose(red[:, 4], ef.sum(1), rtol=1e-5)
    dist.destroy_process_group()


@pytest.mark.parametrize('n,balanced', [(10, False), (11, True), (64, False), (64, True)])
def test_row_shard_plumbing_gloo_world2(n, balanced):
    mp.spawn(_gloo_worker, args=(2, _free_port(), n, balanced), nprocs=2, join=True)


def test_local_csr_of_two_row_ranges():
    """Host side of a sharded plan: the entries of the owned user + item rows in CSR order over the local rows."""
    from sslrec_b200.graph import local_csr
    rs = np.random.RandomState(0)
    n = 50
    rows, cols = rs.randint(0, n, 400), rs.randint(0, n, 400)
    key = np.unique(rows * n + cols)
    rows, cols = key // n, key % n
    perm = rs.permutation(len(rows))
    rows, cols = rows[perm], cols[perm]
    vals = rs.rand(len(rows)).astype(np.float32)
    ranges = ((5, 12), (30, 41))
    rowptr, rows_s, cols_s, vals_s, order = local_csr(rows, cols, vals, ranges)
    owned = list(range(5, 12)) + list(range(30, 41))
    assert rowptr.shape[0] == len(owned) + 1 and rowptr[-1] == len(rows_s)
    for li, r in enumerate(owned):
        seg = slice(rowptr[li], rowptr[li + 1])
        want = np.sort(cols[rows == r])
        assert np.array_equal(cols_s[seg], want) and np.all(rows_s[seg] == r)
    assert np.array_equal(vals[order], vals_s) and np.array_equal(rows[order], rows_s)


def _dp_gloo_worker(rank, world, port):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from sslrec_b200.parallel import BatchShard
    sync = BatchShard(dist, rank, world)
    # two parameters whose gradients are the halves of one flat sink (the embedding table) + a separate one
    flat = torch.arange(12, dtype=torch.float32).view(6, 2) * (rank + 1)
    pu, pi, pw = (torch.nn.Parameter(torch.zeros(4, 2)), torch.nn.Parameter(torch.zeros(2, 2)), torch.nn.Parameter(torch.zeros(3)))
    pu.grad, pi.grad, pw.grad = flat[:4], flat[4:], torch.full((3,), float(rank))
    bufs = sync.coalesce([pi.grad, pw.grad, pu.grad])
    assert sorted(b.numel() for b in bufs) == [3, 12]            # the adjacent halves travel as one buffer
    sync.average_gradients([pu, pi, pw, torch.nn.Parameter(torch.zeros(1))])   # a parameter without .grad is skipped
    want = torch.arange(12, dtype=torch.float32).view(6, 2) * (sum(range(1, world + 1)) / world)
    assert torch.equal(flat, want) and torch.equal(pu.grad, want[:4]) and torch.equal(pi.grad, want[4:])
    assert torch.allclose(pw.grad, torch.full((3,), (world - 1) / 2.0))
    # the loader gives every rank a disjoint share of each epoch
    ds = torch.utils.data.TensorDataset(torch.arange(20))
    loader = sync.shard_loader(ds, batch_size=4, seed=7)
    loader.sampler.set_epoch(3)
    mine = torch.cat([b[0] for b in loader])
    seen = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(seen, mine)
    assert sorted(torch.cat(seen).tolist()) == list(range(20))
    dist.destroy_process_group()


def test_batch_shard_gradient_average_gloo_world2():
    mp.spawn(_dp_gloo_worker, args=(2, _free_port()), nprocs=2, join=True)


def _dp_gpu_worker(rank, world, port, out):
    """Data-parallel step (one batch per rank, averaged gradients) == the single-GPU step on the concatenated batch."""
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
    import ssl_test_helpers as H
    from oracle import inputs, replay
    from sslrec_b200.optim import FusedAdam
    from sslrec_b200.parallel import BatchShard
    for name in ('simgcl', 'lightgcn'):
        g = replay.load_golden(name, 'small')
        case = inputs.make_case('small')
        full = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')]
        half = full[0].numel() // world
        out = {}
        for dp in (False, True):
            model, _ = H.make_model(name, case, g['hp'], device=f'cuda:{rank}')
            model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']})
            opt = FusedAdam(model.parameters(), lr=1e-2)
            batch = [t[rank * half:(rank + 1) * half] for t in full] if dp else [t[:world * half] for t in full]
            loss, _ = model.cal_loss(batch)
            loss.backward()
            if dp:
                BatchShard(dist, rank, world).average_gradients(model.parameters())
                dist.all_reduce(loss, op=dist.ReduceOp.AVG)
            grads = (model.user_embeds.grad.clone(), model.item_embeds.grad.clone())
            opt.step()
            out[dp] = (loss.item(), grads, model.user_embeds.detach().clone(), model.item_embeds.detach().clone())
        assert abs(out[True][0] - out[False][0]) <= 2e-6 * max(1.0, abs(out[False][0])), name
        for a, b in zip(out[True][1], out[False][1]):
            assert torch.allclose(a, b, rtol=1e-4, atol=1e-7 + 2e-5 * b.abs().max().item()), name
        # identical parameters on every rank after the step
        for p in out[True][2:]:
            ref = p.clone()
            dist.broadcast(ref, src=0)
            assert torch.equal(p, ref), name
    dist.destroy_process_group()


@pytest.mark.gpu
def test_data_parallel_step_matches_big_batch():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    mp.spawn(_dp_gpu_worker, args=(2, _free_port(), None), nprocs=2, join=True)


def _gpu_worker(rank, world, port, backend):
    """Row-sharded steps (loss-only sharding; sharded propagation with the fused NVLink stores and with the
    all-gather after the launch) against the single-GPU step: loss, the gradient rows each rank owns, and the parameters
    after Adam.  backend 'nccl': one GPU per rank.  backend 'gloo': every rank on cuda:0 (collectives staged through the
    host) -- the whole sharded path except the peer stores, runnable on a one-GPU machine."""
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    devi = rank if backend == 'nccl' else 0
    torch.cuda.set_device(devi)
    if backend == 'nccl':
        dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', devi))
    else:
        dist.init_process_group('gloo', rank=rank, world_size=world)
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
    import ssl_test_helpers as H
    from oracle import inputs, replay
    from sslrec_b200.optim import FusedAdam
    from sslrec_b200.parallel import RowShard
    case = inputs.make_case('small')
    nu, n = case['n_user'], case['n_user'] + case['n_item']
    for name, gname in (('lightgcn', 'lightgcn'), ('simgcl', 'simgcl'), ('sgl', 'sgl'), ('sgl_nd', 'sgl_nd')):
        size = 'tiny' if name == 'sgl_nd' else 'small'
        g = replay.load_golden(gname, size)
        case = inputs.make_case(size)
        nu, n = case['n_user'], case['n_user'] + case['n_item']
        batch = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')]
        res = {}
        modes = ('single', 'loss', 'symm', 'nccl') if backend == 'nccl' else ('single', 'loss', 'nccl')
        for mode in modes:
            model, _ = H.make_model(name.split('_')[0], case, g['hp'], device=f'cuda:{devi}')
            model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']})
            comm = None
            if mode != 'single':
                ub = ib = None
                if mode == 'nccl':            # unequal blocks balanced by the rows' entry counts (the other modes: equal blocks)
                    from sslrec_b200.parallel import balanced_bounds
                    ub = balanced_bounds(torch.bincount(torch.from_numpy(case['rows']), minlength=nu).float() + 1, world)
                    ib = balanced_bounds(torch.bincount(torch.from_numpy(case['cols']), minlength=n - nu).float() + 1, world)
                comm = RowShard(dist, rank, world, n, n_user=nu, shard_propagation=(mode != 'loss'),
                                transport='nccl' if mode == 'nccl' else 'auto', user_bounds=ub, item_bounds=ib)
                model.shard_to(comm)
            opt = FusedAdam(model.parameters(), lr=1e-2, row_shards=getattr(model, 'row_shards', None), comm=comm)
            losses = []
            for step in range(2):                        # the second step re-uses every shared table
                opt.zero_grad()
                loss, _ = model.cal_loss(batch)
                loss.backward()
                if step == 0:
                    grads = torch.cat([model.user_embeds.grad, model.item_embeds.grad]).clone()
                opt.step()
                losses.append(loss.item())
            torch.cuda.synchronize()
            res[mode] = (losses, grads, torch.cat([model.user_embeds.detach(), model.item_embeds.detach()]).clone(), comm)
        ref = res['single']
        for mode in modes[1:]:
            losses, grads, params, comm = res[mode]
            for a, b in zip(losses, ref[0]):
                assert abs(a - b) <= 2e-6 * max(1.0, abs(b)), (name, mode, losses, ref[0])
            rows = torch.arange(n, device=grads.device)
            if mode != 'loss':                           # sharded propagation: a rank computes the gradient rows it owns
                (u0, u1), (i0, i1) = comm.ranges
                rows = torch.cat([rows[u0:u1], rows[i0:i1]])
            tol = 1e-7 + 2e-5 * ref[1].abs().max().item()
            assert torch.allclose(grads[rows], ref[1][rows], rtol=1e-4, atol=tol), (name, mode)
            # two Adam steps at lr 1e-2.  Adam divides by sqrt(v) + 1e-8: an entry whose gradient is at rounding level (the
            # summation order of the atomics differs between runs) moves by up to ~lr * noise / eps ~ 1e-4, a missed or doubled
            # row update would be off by ~lr = 1e-2
            assert torch.allclose(params, ref[2], rtol=1e-4, atol=3e-4), (name, mode, (params - ref[2]).abs().max().item())
            twin = params.clone()
            dist.broadcast(twin, src=0)
            if mode == 'loss':
                # replicated propagation / BPR / Adam: every rank repeats the same arithmetic, but the BPR backward adds its
                # batch rows with floating-point atomics, so the replicas agree to rounding
                # (amplified by Adam's division where a gradient entry is itself at rounding level), not bit for bit
                assert torch.allclose(params, twin, rtol=0, atol=3e-4), (name, mode, 'replicas diverged', (params - twin).abs().max().item())
            else:
                # sharded propagation: every row has ONE owner that computes it and stores it into all replicas
                assert torch.equal(params, twin), (name, mode, 'replicas diverged')
    dist.destroy_process_group()


@pytest.mark.gpu
def test_sharded_step_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    mp.spawn(_gpu_worker, args=(2, _free_port(), 'nccl'), nprocs=2, join=True)


@pytest.mark.gpu
@pytest.mark.parametrize('world', [2, 3])
def test_sharded_step_matches_single_gpu_ranks_sharing_one_gpu(world):
    """The same equality with every rank on cuda:0 over gloo: runs wherever one GPU is visible."""
    mp.spawn(_gpu_worker, args=(world, _free_port(), 'gloo'), nprocs=world, join=True)
