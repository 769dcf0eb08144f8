"""CPU tier: the N>1 path on the gloo backend, world_size 2.  The sharding
and the single all-reduce of quimb_b200.dist are exercised with a numpy
stand-in for the device contraction (the product has no CPU arithmetic)."""

import os
import sys
import time

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_ranks(target, port, timeout, world=2):
    """Run ``target(rank, world, port, ret)`` in ``world`` spawned processes
    and return ``ret`` (rank -> result).  Asserts that every rank exited 0 within
    ``timeout`` seconds; a rank still running then is killed and reaped."""
    mp.set_start_method("spawn", force=True)
    mgr = mp.Manager()
    ret = mgr.dict()
    procs = [mp.Process(target=target, args=(r, world, port, ret)) for r in range(world)]
    for p in procs:
        p.start()
    deadline = time.monotonic() + timeout
    try:
        for p in procs:
            p.join(timeout=max(0.0, deadline - time.monotonic()))
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
            p.join()
    assert [p.exitcode for p in procs] == [0] * world
    out = dict(ret)
    mgr.shutdown()
    return out


def _np_contract(arrays, inputs, output, optimize):
    from oracle import contract_np as cn
    return torch.from_numpy(np.ascontiguousarray(
        cn.array_contract([np.asarray(a) for a in arrays], inputs, output, "greedy")))


def _worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from quimb_b200 import dist as qd
    rng = np.random.default_rng(0)               # same data on every rank
    a = rng.standard_normal((4, 3, 5)); b = rng.standard_normal((5, 3, 6)); c = rng.standard_normal((6, 4))
    inputs = [("i", "s", "k"), ("k", "s", "l"), ("l", "t")]
    out, mine = qd.contract_sliced([a, b, c], inputs, ("i", "t"), sliced_inds=("s", "k"),
                                   contract_fn=_np_contract)
    ref = np.einsum("isk,ksl,lt->it", a, b, c)
    ok = np.allclose(out.numpy(), ref, atol=1e-12)
    # automatic choice of the sliced indices: at least one slice per rank
    out2, mine2 = qd.contract_sliced([a, b, c], inputs, ("i", "t"), contract_fn=_np_contract)
    ok = ok and np.allclose(out2.numpy(), ref, atol=1e-12) and len(mine2) >= 1
    # tree and slices searched together (auto-hq + width target): every rank
    # searches, rank 0's choice is broadcast; the stand-in executor receives
    # the Tree of the sliced network
    from tests.circuit_util import random_grid_circuit_amplitude
    arrs, ins, outp, amp = random_grid_circuit_amplitude(3, 3, 8, seed=5)

    def _tree_contract(arrays, inputs_, output_, tree_):
        from oracle import contract_np as cn
        nodes = dict(enumerate(arrays))
        inds = dict(enumerate(tree_.inputs))
        for i, j, k, res in tree_.steps:
            nodes[k] = cn.contract_pair(nodes.pop(i), inds[i], nodes.pop(j), inds[j], res)
            inds[k] = res
        (o,) = nodes.values()
        return np.asarray(o)
    out3, mine3 = qd.contract_sliced(arrs, ins, outp, optimize="auto-hq", target_width=6,
                                     contract_fn=_tree_contract)
    ok = ok and abs(complex(out3.numpy()) - amp) < 1e-12 and len(mine3) >= 1
    # units are disjoint and cover everything
    allu = [None] * world
    dist.all_gather_object(allu, mine)
    flat = sorted(u for m in allu for u in m)
    cover = flat == list(range(15))
    ret[rank] = (bool(ok), bool(cover), len(mine))
    dist.destroy_process_group()


def test_slice_parallel_contraction_gloo_world2():
    ret = _run_ranks(_worker, 29500 + (os.getpid() % 2000), timeout=120)
    assert ret[0][0] and ret[1][0]
    assert ret[0][1] and ret[1][1]
    assert ret[0][2] + ret[1][2] == 15 and abs(ret[0][2] - ret[1][2]) <= 1


def test_shard_units_round_robin():
    from quimb_b200 import dist as qd
    assert qd.shard_units(10, 0, 4) == [0, 4, 8]
    assert qd.shard_units(10, 3, 4) == [3, 7]
    assert sorted(sum((qd.shard_units(7, r, 3) for r in range(3)), [])) == list(range(7))
    assert qd.shard_units(2, 5, 8) == []


def _shard_worker(rank, world, port, ret):
    """BondShard on gloo: slabs tile the bond, all_gather_rows reassembles even
    and ragged slabs, and a row-sharded matvec + inner products reproduce the
    unsharded numbers (numpy stand-in for the device kernels)."""
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from quimb_b200.dist import BondShard
    sh = BondShard()
    ok = sh.active and sh.world_size == world
    rng = np.random.default_rng(1)
    for n in (8, 7):                              # even and ragged
        full = torch.from_numpy(rng.standard_normal((n, 5)))
        lo, hi = sh.slab(n)
        got = sh.all_gather_rows(full[lo:hi].clone(), n)
        ok = ok and torch.equal(got, full)
        # sharded y = H x and <x|y>: slab rows of H, full x, one all-reduce
        H = torch.from_numpy(rng.standard_normal((n, n))); H = H + H.T
        x = full[:, 0].clone()
        y_loc = H[lo:hi] @ sh.all_gather_rows(x[lo:hi].reshape(-1, 1).clone(), n).reshape(-1)
        dot = (x[lo:hi] * y_loc).sum().reshape(1)
        sh.all_reduce_(dot)
        ok = ok and abs(float(dot) - float(x @ H @ x)) < 1e-12
    slabs = [sh.slab(11, r) for r in range(world)]
    ok = ok and slabs[0][0] == 0 and slabs[-1][1] == 11 and all(
        slabs[i][1] == slabs[i + 1][0] for i in range(world - 1))
    ret[rank] = bool(ok)
    dist.destroy_process_group()


def test_bond_shard_gloo_world2():
    ret = _run_ranks(_shard_worker, 31500 + (os.getpid() % 2000), timeout=120)
    assert ret[0] and ret[1]


def _boundary_worker(rank, world, port, ret):
    """Two-sided boundary contraction on gloo: rank 0 sweeps in from xmin,
    rank 1 from xmax, one broadcast of each boundary line, every rank does the
    final contraction.  The host layer runs against the ABI emulator (test
    infrastructure); the exchange layer is the real one."""
    import json
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from tests.abi_emulator import emulated_abi
    from quimb_b200 import boundary as bd
    data = np.load(os.path.join(ROOT, "tests", "golden", "boundary.npz"))
    meta = json.load(open(os.path.join(ROOT, "tests", "golden", "boundary.json")))
    ok = True
    with emulated_abi():
        for name in ("peps44", "flat55", "peps35"):
            m = meta[name]
            ts = [(data[f"{name}__t{k}"], r["inds"], tuple(r["site"]), r["layer"])
                  for k, r in enumerate(m["tensors"])]
            for run in (m["runs"][1], m["runs"][3]):
                v = bd.contract_boundary_two_sided(ts, m["Lx"], m["Ly"],
                                                   layer_tags=m["layers"], **run["kw"])
                ref = complex(*run["value"])
                ok = ok and abs(v - ref) <= 1e-10 * abs(ref)
    ret[rank] = bool(ok)
    dist.destroy_process_group()


def test_two_sided_boundary_contraction_gloo_world2():
    ret = _run_ranks(_boundary_worker, 33500 + (os.getpid() % 2000), timeout=240)
    assert ret[0] and ret[1]


def _two_ended_worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from tests.abi_emulator import emulated_abi
    from quimb_b200 import dist as qd
    from oracle import dmrg_np as dm
    ok = True
    with emulated_abi():
        for L, chi, dtype in ((9, 6, "float64"), (12, 5, "complex128"), (2, 3, "float64")):
            sites = dm.mps_rand(L, chi, seed=L, dtype=dtype)
            # each rank only holds its half
            mine = [s if ((i < L // 2) == (rank == 0)) else None for i, s in enumerate(sites)]
            v = qd.mps_norm2_two_ended(mine, shape="lpr").item()
            ref = dm.mps_norm2(sites)
            ok = ok and abs(v - ref) <= 1e-11 * abs(ref)
    ret[rank] = bool(ok)
    dist.destroy_process_group()


def test_two_ended_mps_norm_gloo_world2():
    ret = _run_ranks(_two_ended_worker, 35500 + (os.getpid() % 2000), timeout=240)
    assert ret[0] and ret[1]


def _sharded_lanczos_worker(rank, world, port, ret):
    """Row-sharded device Lanczos (the bond-sharded DMRG eigensolve's solver)
    on gloo: every rank holds a row slab of the operator and of all Krylov
    vectors; inner products are all-reduced, all ranks take the same decisions
    and agree with the dense eigenvalue.  Host layer on the ABI emulator."""
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from tests.abi_emulator import emulated_abi
    import quimb_b200 as qb
    from quimb_b200.dist import BondShard
    ok = True
    with emulated_abi():
        sh = BondShard()
        rng = np.random.default_rng(4)
        n = 301                                      # ragged slabs
        A = rng.standard_normal((n, n))
        H = A + A.T + np.diag(np.linspace(-40, 40, n))
        lo, hi = sh.slab(n)
        Hloc = qb.asarray(H[lo:hi].copy())
        v0 = rng.standard_normal(n)

        def matvec(v_local):
            full = sh.all_gather_rows(v_local.t.reshape(-1, 1), n).reshape(-1)
            return qb.tensordot(Hloc, qb.asarray(full), axes=((1,), (0,)))

        for ncv, tol in ((8, 1e-8), (40, 1e-10)):
            theta, x, info = qb.eigh_lanczos(matvec, qb.asarray(v0[lo:hi].copy()), ncv=ncv,
                                             tol=tol, return_info=True, comm=sh)
            ref = np.linalg.eigvalsh(H)[0]
            ok = ok and abs(theta - ref) < 1e-7 and info["converged"]
            allinfo = [None] * world
            dist.all_gather_object(allinfo, (round(theta, 12), info["nmatvec"], info["restarts"]))
            ok = ok and allinfo[0] == allinfo[1]
            # the local slabs assemble to a normalised eigenvector
            full = sh.all_gather_rows(x.t.reshape(-1, 1), n).reshape(-1).numpy()
            ok = ok and abs(np.linalg.norm(full) - 1) < 1e-10
            ok = ok and np.linalg.norm(H @ full - theta * full) < 1e-5
    ret[rank] = bool(ok)
    dist.destroy_process_group()


def test_sharded_lanczos_gloo_world2():
    ret = _run_ranks(_sharded_lanczos_worker, 37500 + (os.getpid() % 2000), timeout=240)
    assert ret[0] and ret[1]


def test_bond_sharded_dmrg2_gloo_world2_emulated():
    """The whole bond-sharded DMRG2 (ShardedEffHam2 + sharded thick-restart
    Lanczos + replicated SVD / environments) on gloo with two ranks: energies
    equal the unsharded run and exact diagonalisation, states bit-identical on
    both ranks.  Host layer on the ABI emulator, exchange layer real."""
    from tests.test_gpu_p2p import run_process_group, torchrun_cmd
    rc, out, err = run_process_group(
        torchrun_cmd("dist_dmrg_worker.py", 2, "--backend", "gloo", "--emulate",
                     "--L", "10", "--chi", "20"), timeout=600)
    assert rc == 0 and "DIST_DMRG_OK" in out, out[-2000:] + err[-2000:]
