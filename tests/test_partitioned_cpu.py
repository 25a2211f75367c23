"""Host logic of the row-partitioned path (SURVEY.md 8e "row-sharded variant"), on CPU:
the moment merge against the oracle, the gloo world-2 collectives of the merge operators and the
row-slab -> column-block all-to-all.  No kernels run here."""
import os
import socket

import numpy as np
import pytest
import torch.multiprocessing as mp

from anovos_b200 import engine, partitioned
from oracle import spark_semantics as S


def _record(x):
    """Moment record of one partition, computed by the oracle (float64 on double(x))."""
    r = np.zeros(1, dtype=engine._MOM_DT)
    x = np.asarray(x, dtype=np.float64)
    r["n_valid"], r["n_nonzero"] = x.size, int(np.count_nonzero(x))
    if x.size:
        n, mean, m2, m3, m4 = S.central_moments(x)
        r["min"], r["max"], r["mean"], r["m2"], r["m3"], r["m4"] = x.min(), x.max(), mean, m2, m3, m4
    else:
        r["min"] = r["max"] = r["mean"] = np.nan
    return r


@pytest.mark.parametrize("splits", [[0.5], [0.1, 0.3, 0.9], [0.0, 0.5], [0.25, 0.25, 1.0]])
def test_merge_moments_matches_whole(splits):
    rng = np.random.default_rng(5)
    cols = [rng.normal(1e4, 3.0, 20000), np.exp(rng.normal(0, 0.75, 20000)),
            np.where(rng.random(20000) < 0.7, 0.0, rng.exponential(2.0, 20000))]
    whole = np.concatenate([_record(c) for c in cols])
    cuts = [0] + [int(s * 20000) for s in splits] + [20000]     # includes EMPTY partitions
    parts = [np.concatenate([_record(c[a:b]) for c in cols]) for a, b in zip(cuts[:-1], cuts[1:])]
    got = partitioned.merge_moments(parts)
    assert np.array_equal(got["n_valid"], whole["n_valid"]) and np.array_equal(got["n_nonzero"], whole["n_nonzero"])
    assert np.array_equal(got["min"], whole["min"]) and np.array_equal(got["max"], whole["max"])
    for f in ("mean", "m2", "m3", "m4"):
        np.testing.assert_allclose(got[f], whole[f], rtol=1e-9, err_msg=f)


def test_merge_moments_nan_ordering():
    a, b = _record([1.0, 2.0]), _record([3.0])
    b["max"] = np.nan                      # a partition holding a NaN value: Spark's max is NaN, min ignores it
    m = partitioned.merge_moments([a, b])
    assert np.isnan(m["max"][0]) and m["min"][0] == 1.0
    e = _record([])
    m = partitioned.merge_moments([e, a, e])
    assert m["n_valid"][0] == 2 and m["min"][0] == 1.0 and m["max"][0] == 2.0 and m["mean"][0] == 1.5


def test_merge_moments_all_nan_partition_adds_no_extrema():
    """A partition of nothing but NaN has min = max = NaN (finalize_moments): the merged extrema are those of the
    other partitions, as over the frame held whole; all partitions all-NaN give NaN."""
    a, b = _record([1.0, 2.0]), _record([np.nan, np.nan])
    assert np.isnan(b["min"][0]) and np.isnan(b["max"][0])
    for parts in ([a, b], [b, a], [b, a, b]):
        m = partitioned.merge_moments(parts)
        assert m["min"][0] == 1.0 and m["max"][0] == 2.0
        assert m["n_valid"][0] == sum(int(p["n_valid"][0]) for p in parts)
    m = partitioned.merge_moments([b, b])
    assert np.isnan(m["min"][0]) and np.isnan(m["max"][0])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _table(n, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 1, n).astype(np.float32)
    y = rng.integers(-5, 5, n).astype(np.int64)
    z = rng.integers(0, 3, n).astype(np.int32)
    vy = rng.random(n) > 0.2
    return x, y, vy, z


def _worker(rank, world, port, ret):
    import torch
    import torch.distributed as dist
    from anovos_b200.frame import ColumnFrame, _pack_validity
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    g = partitioned._Group(True)
    # merge operators across ranks
    rec = _record(np.arange(10.0) + 100 * rank)
    allrec = g.all_gather_records(rec)
    merged = partitioned.merge_moments(allrec)
    counts = g.all_reduce(np.array([[1, 2, 3]], np.uint64) * np.uint64(rank + 1))
    regs = g.all_reduce(np.array([rank, 5 - rank, 7], np.uint32), op="max")
    t = torch.arange(4, dtype=torch.int64) * (rank + 1)
    g.all_reduce_device(t)
    # row slabs (64 rows on rank 0, 45 on rank 1) of 4 columns -> column blocks (2 + 2)
    n = 64 if rank == 0 else 45
    x, y, vy, z = _table(n, 10 + rank)
    fr = ColumnFrame.from_tensors({"x": x, "y": (y, _pack_validity(vy)), "z": (z, None, ["a", "b", "c"]), "w": x * 2})
    out = partitioned.repartition_to_columns(fr, True)
    got = {}
    for name in out.columns:
        c = out.column(name)
        got[name] = (np.array(c._host), None if c._host_valid is None else np.array(c._host_valid), c.dictionary)
    ret[rank] = dict(merged=merged.tolist(), counts=counts.tolist(), regs=regs.tolist(), t=t.tolist(), cols=got,
                     n_rows=out.n_rows)
    dist.destroy_process_group()


def test_row_slab_collectives_and_repartition_world2():
    from anovos_b200.frame import _pack_validity
    world, port = 2, _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    a, b = ret[0], ret[1]
    whole = _record(np.concatenate([np.arange(10.0), np.arange(10.0) + 100]))
    assert a["merged"] == b["merged"]
    np.testing.assert_allclose(np.array(a["merged"][0][4:]), np.array(whole.tolist()[0][4:]), rtol=1e-12)
    assert a["counts"] == [[3, 6, 9]] and a["regs"] == [1, 5, 7] and a["t"] == [0, 3, 6, 9]
    # rank 0 owns x, y ; rank 1 owns z, w - each holding all 109 rows in slab order
    assert a["n_rows"] == b["n_rows"] == 109
    assert sorted(a["cols"]) == ["x", "y"] and sorted(b["cols"]) == ["w", "z"]
    x0, y0, vy0, z0 = _table(64, 10)
    x1, y1, vy1, z1 = _table(45, 11)
    assert np.array_equal(a["cols"]["x"][0], np.concatenate([x0, x1])) and a["cols"]["x"][1] is None
    assert np.array_equal(a["cols"]["y"][0], np.concatenate([y0, y1]))
    assert np.array_equal(np.asarray(a["cols"]["y"][1]).view(np.uint32),
                          np.asarray(_pack_validity(np.concatenate([vy0, vy1]))).view(np.uint32))
    assert np.array_equal(b["cols"]["z"][0], np.concatenate([z0, z1])) and b["cols"]["z"][2] == ["a", "b", "c"]
    assert np.array_equal(b["cols"]["w"][0], np.concatenate([x0 * 2, x1 * 2]))
