"""cat_to_num_supervised on a PartitionedFrame whose row slabs sit on two ranks (gloo world 2, NumPy kernel stand-ins):
every rank fits the same model as the oracle on the whole table.  The event rows of the null group and all event rows
of one category sit on rank 1 only, so a count taken over the local slab instead of the group shows up in the rates."""
import os
import socket

import numpy as np
import pyarrow as pa
import torch.multiprocessing as mp

import encoding_oracle as E

DIC = ["a", "b", "c"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _slab(rank):
    """(codes, valid, label) of the rank's 70 (rank 0) or 45 (rank 1) rows; rank 0 holds no event row."""
    n = 70 if rank == 0 else 45
    rng = np.random.default_rng(20 + rank)
    codes = rng.integers(0, 3, n).astype(np.int32)
    valid = rng.random(n) > 0.25
    label = np.zeros(n, np.int32) if rank == 0 else (rng.random(n) > 0.4).astype(np.int32)
    if rank == 1:
        label[~valid] = 1                      # the null group's event rows live here
    return codes, valid, label


def _worker(rank, world, port, ret):
    import torch.distributed as dist
    from anovos_b200.frame import ColumnFrame, _pack_validity
    from anovos_b200.partitioned import PartitionedFrame
    from test_encoding_cpu import stand_ins
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    codes, valid, label = _slab(rank)
    with stand_ins():
        import anovos.data_transformer.transformers as T
        fr = ColumnFrame.from_tensors({"c": (codes, _pack_validity(valid), DIC), "y": label})
        half = 32
        pf = PartitionedFrame.from_frames([fr.slice_rows(0, half), fr.slice_rows(half, fr.n_rows)], group=True)
        odf = T.cat_to_num_supervised(None, pf, list_of_cols=["c"], label_col="y", event_label=1, output_mode="append")
        ret[rank] = pa.concat_tables([ch.to_arrow() for ch in odf.chunks()]).column("c_encoded").to_pylist()
    dist.destroy_process_group()


def test_supervised_rates_over_row_slabs_world2():
    world, port = 2, _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    parts = [_slab(r) for r in range(world)]
    codes = np.concatenate([p[0] for p in parts])
    valid = np.concatenate([p[1] for p in parts])
    label = np.concatenate([p[2] for p in parts])
    table = pa.table({"c": pa.array([DIC[k] if ok else None for k, ok in zip(codes, valid)]), "y": pa.array(label)})
    exp, models = E.cat_to_num_supervised(table, list_of_cols=["c"], label_col="y", event_label=1, output_mode="append")
    assert models["c"][0][0] is None and models["c"][0][1] > 0      # the null group has event rows (all on rank 1)
    col = exp.column("c_encoded").to_pylist()
    assert ret[0] + ret[1] == col
