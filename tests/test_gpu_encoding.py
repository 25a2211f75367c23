"""The categorical encoders on the GPU: anv_code_map and anv_one_hot bit for bit against NumPy on adversarial columns,
and cat_to_num_unsupervised / cat_to_num_supervised / outlier_categories against the oracle (tests/encoding_oracle.py)
on the Spark-partitioned income table, on 10 M-row synthetic frames and on chunked frames."""
import warnings

import numpy as np
import pyarrow as pa
import pytest

import encoding_oracle as E
from test_encoding_cpu import same_tables

pytestmark = pytest.mark.gpu


def _words(valid):
    bits = np.packbits(np.asarray(valid, bool), bitorder="little")
    return np.concatenate([bits, np.zeros((-len(bits)) % 4, np.uint8)]).view(np.int32)


def _frame(cols):
    """name -> (codes int32, bool valid | None, dictionary) -> device-resident ColumnFrame."""
    import torch
    from anovos_b200.frame import ColumnFrame
    return ColumnFrame.from_tensors({n: (torch.from_numpy(np.ascontiguousarray(v)).cuda(),
                                         None if ok is None else torch.from_numpy(_words(ok)).cuda(), dic)
                                     for n, (v, ok, dic) in cols.items()})


def _slots(codes, ok, size):
    """The slot every row reads: min((uint32)code, size) for a valid row, size for a null one."""
    s = np.minimum(codes.astype(np.int64) & 0xFFFFFFFF, size)
    return np.where(ok, s, size)


def _columns(n, size, rng):
    """Codes of a dictionary of `size`, with codes outside it (negative and past the end) written through the C ABI."""
    codes = rng.integers(0, max(size, 1), n).astype(np.int32)
    bad = rng.random(n) < 0.05
    codes[bad] = rng.choice(np.array([-1, -(1 << 31), size, size + 7, (1 << 31) - 1], np.int32), int(bad.sum()))
    dic = ["k%d" % i for i in range(size)]
    lead_null = np.ones(n, bool)
    lead_null[:min(n, 66_000)] = False
    return {"some": (codes, rng.random(n) > 0.3, dic), "free": (codes, None, dic), "all_null": (codes, np.zeros(n, bool), dic),
            "lead_null": (codes, lead_null, dic)}


@pytest.mark.parametrize("n", [1, 5, 31, 33, 130, 1027, 70_001])
@pytest.mark.parametrize("size", [0, 1, 10_000])
def test_code_map_bit_exact(n, size):
    from anovos_b200 import engine
    rng = np.random.default_rng([n, size])
    cols = _columns(n, size, rng)
    names, tables, evs = [], [], []
    for name in cols:
        ti = rng.integers(-(1 << 31), (1 << 31) - 1, size + 1).astype(np.int32)
        td = rng.normal(0, 1, size + 1) * 10.0 ** rng.integers(-300, 300, size + 1)
        td[:min(size + 1, 2)] = [np.nan, -0.0][:min(size + 1, 2)]
        for t in (ti, td):
            for ev in (None, rng.random(size + 1) > 0.4):
                names.append(name)
                tables.append(t)
                evs.append(ev)
    fr = _frame(cols)
    outs, valid, nulls = engine.code_map(fr, names, tables, evs)
    for i, (name, t, ev) in enumerate(zip(names, tables, evs)):
        codes, ok, _ = cols[name]
        s = _slots(codes, np.ones(n, bool) if ok is None else ok, size)
        exp = t[s]
        got = outs[i].cpu().numpy()
        if ev is None:
            assert valid[i] is None and nulls[i] == 0
        else:
            keep = ev[s]
            exp = np.where(keep, exp, t.dtype.type(0))
            assert np.array_equal(valid[i].cpu().numpy(), _words(keep)[:(n + 31) // 32]), (name, n)
            assert nulls[i] == int((~keep).sum())
        assert got.dtype == exp.dtype and np.array_equal(got.view(np.uint8), exp.view(np.uint8)), (name, n, t.dtype)


@pytest.mark.parametrize("n", [1, 6, 33, 1027, 70_001])
@pytest.mark.parametrize("size,k", [(0, 1), (1, 2), (9, 10), (50, 51), (1024, 1025), (10_000, 17)])
def test_one_hot_bit_exact(n, size, k):
    from anovos_b200 import engine
    rng = np.random.default_rng([n, size, k])
    cols = _columns(n, size, rng)
    idx = rng.integers(0, k, size + 1).astype(np.int32)
    idx[rng.random(size + 1) < 0.1] = k + 3                  # an entry outside [0, k) sets no output
    outs = engine.one_hot(_frame(cols), list(cols), [idx] * len(cols), [k] * len(cols))
    stride = engine.one_hot_stride(n)
    for o, (name, (codes, ok, _)) in zip(outs, cols.items()):
        s = _slots(codes, np.ones(n, bool) if ok is None else ok, size)
        exp = (idx[s][None, :] == np.arange(k)[:, None]).astype(np.int32)
        assert o.shape == (k, n) and o.stride(0) == stride
        assert all(o[j].data_ptr() % 16 == 0 for j in range(min(k, 3)))
        assert np.array_equal(o.cpu().numpy(), exp), (name, n, k)
        base = o.as_strided((k, stride), (stride, 1)).cpu().numpy()
        assert not base[:, n:].any()                          # the padding rows are zero


def test_wide_calls_run_in_column_blocks():
    from anovos_b200 import engine
    n, m = 37, 65_538
    rng = np.random.default_rng(5)
    codes = rng.integers(0, 3, n).astype(np.int32)
    ok = rng.random(n) > 0.2
    fr = _frame({"c": (codes, ok, ["a", "b", "c"])})
    tables = [np.array([i, i + 1, i + 2, -i], np.int32) for i in range(m)]
    outs, valid, nulls = engine.code_map(fr, ["c"] * m, tables, [None] * m)
    got = np.stack([o.cpu().numpy() for o in (outs[0], outs[m // 2], outs[-1])])
    s = _slots(codes, ok, 3)
    assert np.array_equal(got, np.stack([tables[i][s] for i in (0, m // 2, m - 1)]))
    assert len(outs) == m and not nulls.any()
    idx = [np.array([i % 2, 1 - i % 2, 0, 1], np.int32) for i in range(m)]
    oh = engine.one_hot(fr, ["c"] * m, idx, [2] * m)
    for i in (0, 65_535, m - 1):
        assert np.array_equal(oh[i].cpu().numpy(), (idx[i][s][None] == np.arange(2)[:, None]).astype(np.int32))


# ---- the API against the oracle -------------------------------------------------------------------------------------

def _product(name, frame, **kw):
    import anovos.data_transformer.transformers as T
    odf = getattr(T, name)(None, frame, **kw)
    if getattr(odf, "is_partitioned", False):
        return pa.concat_tables([ch.to_arrow() for ch in odf.chunks()])
    return odf.to_arrow()


CATS = ["workclass", "education", "marital-status", "relationship", "race", "sex", "empty", "geohash"]


@pytest.mark.parametrize("method,order", [("label_encoding", "frequencyDesc"), ("label_encoding", "alphabetAsc"),
                                          ("label_encoding", "frequencyAsc"), ("onehot_encoding", "frequencyDesc")])
@pytest.mark.parametrize("output_mode", ["replace", "append"])
def test_unsupervised_on_partitioned_income(income_spark, income, method, order, output_mode):
    kw = dict(list_of_cols=CATS, method_type=method, index_order=order, cardinality_threshold=100, output_mode=output_mode)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = _product("cat_to_num_unsupervised", income_spark, **kw)
    same_tables(got, E.cat_to_num_unsupervised(income, **kw)[0])


@pytest.mark.parametrize("output_mode", ["replace", "append"])
def test_supervised_and_outliers_on_partitioned_income(income_spark, income, output_mode):
    kw = dict(list_of_cols=CATS, label_col="income", event_label=">50K", output_mode=output_mode)
    same_tables(_product("cat_to_num_supervised", income_spark, **kw), E.cat_to_num_supervised(income, **kw)[0])
    for cov, mx in ((1.0, 10), (0.9, 50), (1.0, 15)):
        kw = dict(list_of_cols=CATS, coverage=cov, max_category=mx, output_mode=output_mode)
        same_tables(_product("outlier_categories", income_spark, **kw), E.outlier_categories(income, **kw)[0])


def test_chunked_frames_equal_resident(income):
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.partitioned import PartitionedFrame
    res = ColumnFrame.from_arrow(income)
    part = PartitionedFrame.from_frame(income, 4096)
    for name, kw in [("cat_to_num_unsupervised", dict(method_type="onehot_encoding", cardinality_threshold=60)),
                     ("cat_to_num_unsupervised", dict(index_order="alphabetDesc")),
                     ("cat_to_num_supervised", dict(label_col="income", event_label="<=50K")),
                     ("outlier_categories", dict(coverage=0.8))]:
        same_tables(_product(name, part, **kw), _product(name, res, **kw))


def _labels_np(codes, ok, dic):
    cnt = np.bincount(codes[ok], minlength=len(dic))
    present = [k for k in range(len(dic)) if cnt[k]]
    return sorted(present, key=lambda k: (-int(cnt[k]), dic[k].encode())), cnt


def test_synthetic_10m_rows_against_numpy():
    """The four cardinalities at 10 M rows: label encoding (the 10 000-key column included), supervised encoding with the
    card-2 column as the label, one-hot of the card-12 column, all against NumPy images of the semantics."""
    import anovos.data_transformer.transformers as T
    from anovos_b200 import synth
    from anovos_b200.shared.utils import spark_round
    n = 10_000_000
    fr = synth.device_frame(n, 4, seed=11, cat_every=1)
    names = fr.columns
    host = {}
    for c in names:
        d, v = fr.column(c).device()
        ok = np.ones(n, bool) if v is None else np.unpackbits(v.cpu().numpy().view(np.uint8), bitorder="little")[:n] > 0
        host[c] = (d.cpu().numpy(), ok, fr.column(c).dictionary)
    cards = sorted(names, key=lambda c: len(host[c][2]))
    lab_col, c12, c10k = cards[0], cards[1], cards[-1]

    odf = T.cat_to_num_unsupervised(None, fr, list_of_cols=names, cardinality_threshold=20_000)
    for c in names:
        codes, ok, dic = host[c]
        order, _ = _labels_np(codes, ok, dic)
        pos = np.full(len(dic), len(order), np.int32)
        pos[order] = np.arange(len(order), dtype=np.int32)
        d, v = odf.column(c).device()
        assert np.array_equal(d.cpu().numpy()[ok], pos[codes[ok]]), c
        if v is None:
            assert ok.all(), c
        else:
            assert np.array_equal(np.unpackbits(v.cpu().numpy().view(np.uint8), bitorder="little")[:n] > 0, ok), c
        assert odf.column(c).sdtype == "int"

    oh = T.cat_to_num_unsupervised(None, fr, list_of_cols=[c12], method_type="onehot_encoding")
    codes, ok, dic = host[c12]
    order, _ = _labels_np(codes, ok, dic)
    pos = np.full(len(dic), len(order), np.int32)
    pos[order] = np.arange(len(order), dtype=np.int32)
    idx = np.where(ok, pos[np.where(ok, codes, 0)], len(order))
    for j in range(len(order) + 1):
        assert np.array_equal(oh.column("%s_%d" % (c12, j)).device()[0].cpu().numpy(), (idx == j).astype(np.int32)), j

    ev_code = host[lab_col][2][0]
    sup = T.cat_to_num_supervised(None, fr, list_of_cols=[c10k, c12], label_col=lab_col, event_label=ev_code)
    lc, lok, _ = host[lab_col]
    is_ev = lok & (lc == 0)
    for c in (c10k, c12):
        codes, ok, dic = host[c]
        g = np.where(ok, codes + 1, 0)
        tot = np.bincount(g, minlength=len(dic) + 1)
        e = np.bincount(g[is_ev], minlength=len(dic) + 1)
        rate = np.array([spark_round(e[k] / tot[k], 4) if tot[k] else 0.0 for k in range(len(dic) + 1)])
        d, v = sup.column(c).device()
        bits = np.unpackbits(v.cpu().numpy().view(np.uint8), bitorder="little")[:n] > 0
        assert np.array_equal(bits, ok), c
        assert np.array_equal(d.cpu().numpy()[ok], rate[g[ok]]), c
