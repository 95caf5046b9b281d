"""world_size-2 gloo tests (CPU) of the multi-GPU exchange logic in arrow_b200.distributed:
row-range shards -> local pass -> one all-to-all -> merge must reproduce the single-process oracle."""
import os
import socket
import sys

import numpy as np
import pyarrow as pa
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0x0FF1CE


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _data(n):
    rng = np.random.default_rng(SEED)
    keys = pa.array(rng.integers(0, 500, n, dtype=np.int64), mask=rng.random(n) < 0.03)
    vals = pa.array(rng.integers(-100, 100, n, dtype=np.int64), mask=rng.random(n) < 0.1)
    sortkeys = pa.array(rng.integers(-2**40, 2**40, n, dtype=np.int64), mask=rng.random(n) < 0.1)
    dup = pa.array(rng.integers(0, 20, n, dtype=np.int64), mask=rng.random(n) < 0.1)  # many ties: stability
    return keys, vals, sortkeys, dup


# Valid rows 1 (mod 10) only: with 10 000-row shards and 1000 samples per rank, every row on an evenly spaced grid over the
# whole shard is null, so a sampler that does not look among the valid rows finds no splitter at all.
SPARSE_ROWS, SPARSE_SAMPLES = 20000, 1000


def _sparse():
    valid = np.arange(SPARSE_ROWS) % 10 == 1
    return pa.array(np.arange(SPARSE_ROWS, 0, -1, dtype=np.int64), mask=~valid)


# the null key's partial sum on rank 0 is >= 2^63: it must travel as its bits, not as an int64 value
U64_KEYS = pa.array([None, None, 1, 2], pa.int64())
U64_VALS = pa.array([2**63 + 5, 3, 7, 9], pa.uint64())


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from arrow_b200 import distributed as d  # imports the module only (no CUDA library needed for HostOps)
    from tests.host_ops import HostOps
    ops = HostOps()
    n = 20001
    keys, vals, sortkeys, dup = _data(n)
    lo, hi = rank * n // world, (rank + 1) * n // world
    k, s, c = d.group_by_sum_count(keys.slice(lo, hi - lo), vals.slice(lo, hi - lo), ops, d.TorchExchange())
    res = {"k": k.to_pylist(), "s": s.to_pylist(), "c": c.to_pylist()}
    for name, col in (("wide", sortkeys), ("dup", dup)):
        seg, nulls = d.sort_indices(col.slice(lo, hi - lo), ops, d.TorchExchange(), samples_per_rank=64)
        res[name] = (seg.tolist(), nulls.tolist())
    lo, hi = rank * SPARSE_ROWS // world, (rank + 1) * SPARSE_ROWS // world
    seg, nulls = d.sort_indices(_sparse().slice(lo, hi - lo), ops, d.TorchExchange(), samples_per_rank=SPARSE_SAMPLES)
    res["sparse"] = (seg.tolist(), nulls.tolist())
    lo, hi = rank * len(U64_KEYS) // world, (rank + 1) * len(U64_KEYS) // world
    k, s, c = d.group_by_sum_count(U64_KEYS.slice(lo, hi - lo), U64_VALS.slice(lo, hi - lo), ops, d.TorchExchange())
    res["u64"] = list(zip(k.to_pylist(), s.to_pylist(), c.to_pylist()))
    torch.save(res, os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_exchange_logic_world2(tmp_path):
    from oracle import arrow_oracle as ora
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(os.path.join(tmp_path, f"r{r}.pt")) for r in range(world)]
    n = 20001
    keys, vals, sortkeys, dup = _data(n)
    # group-by: owners are disjoint, union == the single-process answer (compared sorted by key)
    uniq, (s, c) = ora.group_by([keys], [("hash_sum", vals, None), ("hash_count", vals, None)])
    want = sorted(zip(uniq[0].to_pylist(), s.to_pylist(), c.to_pylist()), key=lambda t: (t[0] is None, t[0]))
    got = sorted([t for r in res for t in zip(r["k"], r["s"], r["c"])], key=lambda t: (t[0] is None, t[0]))
    assert got == want
    owned = [set(r["k"]) for r in res]
    assert not (owned[0] & owned[1])
    # sort: rank-ordered concatenation of value segments, then of null segments == stable sort_indices
    for name, col in (("wide", sortkeys), ("dup", dup)):
        cat = [i for r in res for i in r[name][0]] + [i for r in res for i in r[name][1]]
        assert cat == ora.sort_indices(col).to_pylist(), name
        assert all(len(r[name][0]) > 0 for r in res)  # splitters balanced the ranks
    cat = [i for r in res for i in r["sparse"][0]] + [i for r in res for i in r["sparse"][1]]
    assert cat == ora.sort_indices(_sparse()).to_pylist(), "sparse valid rows"
    assert all(len(r["sparse"][0]) > 0 for r in res)
    got = sorted([t for r in res for t in r["u64"]], key=lambda t: (t[0] is None, t[0]))
    assert got == [(1, 7, 1), (2, 9, 1), (None, 2**63 + 8, 2)]
