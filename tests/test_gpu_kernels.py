"""GPU parity tests of the raw kernels (through the C-ABI) against the oracle."""
import math

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu

from oracle import spark_semantics as S


def _mixed_table(n, seed=0, null_rate=0.1):
    rng = np.random.default_rng(seed)
    def mask():
        return rng.random(n) < null_rate
    cols = {
        "f32_norm": pa.array((rng.normal(1000.0, 3.0, n)).astype(np.float32), mask=mask()),
        "f32_logn": pa.array(np.exp(rng.normal(0, 0.75, n)).astype(np.float32)),
        "f32_zero": pa.array(np.where(rng.random(n) < 0.7, 0.0, rng.exponential(2.0, n)).astype(np.float32), mask=mask()),
        "f64_unif": pa.array(rng.uniform(-5, 12, n), mask=mask()),
        "i32": pa.array(rng.integers(-50, 1000, n).astype(np.int32), mask=mask()),
        "i64": pa.array(rng.integers(-10**12, 10**12, n).astype(np.int64)),
        "f32_allnull": pa.array(np.zeros(n, np.float32), mask=np.ones(n, bool)),
        "f32_const": pa.array(np.full(n, 3.25, np.float32)),
    }
    return pa.table(cols)


@pytest.mark.parametrize("n", [1, 5, 33, 1000, 16384 + 7, 300001])
def test_moments_vs_oracle(n):
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    t = _mixed_table(n, seed=n)
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    m = engine.moments(fr, names)
    for i, c in enumerate(names):
        vals, valid = S.column_values(t, c)
        x = vals[valid].astype(np.float64)
        nn, mean, m2, m3, m4 = S.central_moments(x)
        assert m["n_valid"][i] == nn, c                                   # bit-exact counts
        assert m["n_nonzero"][i] == int(np.count_nonzero(x != 0)), c
        if nn == 0:
            assert math.isnan(m["min"][i]) and math.isnan(m["max"][i])
            continue
        assert m["min"][i] == x.min() and m["max"][i] == x.max(), c      # bit-exact extrema
        scale = max(abs(mean), math.sqrt(m2 / nn), 1e-300)
        assert abs(m["mean"][i] - mean) <= 1e-9 * scale, c
        for k, (g, e) in enumerate(((m["m2"][i], m2), (m["m3"][i], m3), (m["m4"][i], m4))):
            tol = 1e-6 * abs(e) + 1e-9 * (m2 / nn) ** ((k + 2) / 2) * nn   # 1e-6 relative (north_star)
            assert abs(g - e) <= tol, (c, k + 2, g, e)


@pytest.mark.parametrize("bins", [2, 10, 20, 39, 64, 300])
def test_histogram_bit_exact(bins):
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    n = 200003
    t = _mixed_table(n, seed=bins).drop_columns(["f32_allnull"])
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    mom = engine.moments(fr, names)
    cuts, lohi = [], []
    for i, c in enumerate(names):
        mn, mx = float(mom["min"][i]), float(mom["max"][i])
        cuts.append(S.equal_range_cutoffs(mn, mx, bins))
        lohi.append((mn, mx))
    model = engine.BinModel(fr, names, cuts, lohi)
    assert model.specs_host["mode"][names.index("f32_logn")] == 1
    assert model.specs_host["mode"][names.index("f32_const")] == 0   # degenerate range -> generic path
    h = engine.histogram(fr, model)
    m2, h2 = engine.moments_histogram(fr, model)
    assert (h == h2).all()
    for f in engine.MOMENT_FIELDS:
        assert np.array_equal(mom[f], m2[f], equal_nan=True), f
    ids = engine.bin_assign(fr, model).cpu().numpy()
    for i, c in enumerate(names):
        vals, valid = S.column_values(t, c)
        exp = S.assign_bins(vals, valid, cuts[i], bins)   # integer columns compare exactly
        assert np.array_equal(ids[i], exp), c                              # bit-exact bin ids
        cnt = np.bincount(exp, minlength=bins + 1)
        assert np.array_equal(h[i, :bins + 1], cnt.astype(np.uint64)), c   # bit-exact counts


def test_histogram_generic_cutoffs_with_duplicates():
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    n = 100000
    t = _mixed_table(n, seed=7).select(["f32_zero", "f32_norm", "i32", "f64_unif"])
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    cuts = []
    for c in names:
        vals, valid = S.column_values(t, c)
        srt = np.sort(vals[valid].astype(np.float64))
        cuts.append(S.equal_frequency_cutoffs(srt, 10))
    assert len(set(cuts[0])) < 9  # zero-inflated: duplicated cutoffs
    model = engine.BinModel(fr, names, cuts, None)
    h = engine.histogram(fr, model)
    for i, c in enumerate(names):
        vals, valid = S.column_values(t, c)
        exp = S.assign_bins(vals, valid, cuts[i], 10)
        assert np.array_equal(h[i, :11], np.bincount(exp, minlength=11).astype(np.uint64)), c


def test_code_counts_and_drift_reduce():
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    rng = np.random.default_rng(3)
    n = 120000
    cats = {}
    for card in (2, 12, 100, 12000):
        dic = np.array(["cat_%05d" % i for i in range(card)], dtype=object)
        codes = np.minimum((rng.pareto(1.2, n)).astype(np.int64), card - 1)
        cats["c%d" % card] = pa.array(dic[codes], mask=rng.random(n) < 0.05)
    t = pa.table(cats)
    fr = ColumnFrame.from_arrow(t)
    counts = engine.code_counts(fr, t.column_names)
    for c, h in zip(t.column_names, counts):
        col = fr.column(c)
        vals, valid = S.column_values(t, c)
        assert h[0] == int((~valid).sum())
        u, k = np.unique(vals[valid].astype(str), return_counts=True)
        got = {col.dictionary[i]: int(h[i + 1]) for i in range(len(col.dictionary)) if h[i + 1]}
        assert got == dict(zip(u.tolist(), k.tolist())), c
    # drift reduce vs the oracle's sequential loop
    src = [np.array([5, 0, 10, 20, 0, 7], np.uint64), np.array([0, 3, 3, 0], np.uint64), np.array([2, 0, 9], np.uint64)]
    tgt = [np.array([0, 4, 0, 25, 0, 9], np.uint64), np.array([0, 3, 3, 0], np.uint64), np.array([1, 4, 9], np.uint64)]
    kinds = [0, 0, 1]
    # wide tables (string columns with many keys) take the CTA-per-column path: keys missing on either side,
    # null groups on none / one / both sides, a table exactly one key past the narrow limit
    for width, nulls_s, nulls_t, kind in ((97, 0, 0, 1), (5000, 3, 0, 1), (12001, 4, 9, 1), (300, 1, 1, 0)):
        a = rng.integers(0, 50, width + 1).astype(np.uint64) * (rng.random(width + 1) < 0.8)
        b = rng.integers(0, 50, width + 1).astype(np.uint64) * (rng.random(width + 1) < 0.8)
        a[0], b[0] = nulls_s, nulls_t
        src.append(a.astype(np.uint64))
        tgt.append(b.astype(np.uint64))
        kinds.append(kind)
    ns, nt = 4200000, 3800000
    d = engine.drift_reduce(src, tgt, kinds, ns, nt)
    for i in range(len(src)):
        sg = {k: int(v) for k, v in enumerate(src[i]) if k and v}
        tg = {k: int(v) for k, v in enumerate(tgt[i]) if k and v}
        nulls = 0
        if kinds[i] == 0:
            if src[i][0]:
                sg[-1] = 0
            if tgt[i][0]:
                tg[-1] = 0
        else:
            nulls = int(src[i][0] > 0) + int(tgt[i][0] > 0)
        keys = sorted(set(sg) | set(tg))
        e = S.drift_from_groups(sg, tg, ns, nt, keys, nulls)
        for g, ev in zip((d["psi"][i], d["hd"][i], d["jsd"][i], d["ks"][i]), e):
            assert abs(g - ev) <= 1e-12 * max(1.0, abs(ev)), (i, g, ev)


def test_synth_generator_reproducible_and_sane():
    import ctypes as C
    import torch
    from anovos_b200 import _lib, engine
    L = _lib.lib()
    n = 1000003
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    outs = []
    for rep in range(2):
        x = torch.empty(n, dtype=torch.float32, device="cuda")
        v = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
        _lib.check(L.anv_synth_f32(x.data_ptr(), v.data_ptr(), n, 42, 3, 0, 5.0, 2.0, 0.02, st))
        outs.append((x.cpu().numpy(), v.cpu().numpy()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    x, v = outs[0]
    valid = np.unpackbits(v.view(np.uint8), bitorder="little")[:n].astype(bool)
    assert abs(valid.mean() - 0.98) < 2e-3
    assert abs(x.mean() - 5.0) < 0.02 and abs(x.std() - 2.0) < 0.02
    c = torch.empty(n, dtype=torch.int32, device="cuda")
    _lib.check(L.anv_synth_codes(c.data_ptr(), None, n, 42, 9, 100, 1.2, 0.0, st))
    cc = c.cpu().numpy()
    assert cc.min() == 0 and cc.max() <= 99 and np.bincount(cc)[0] > np.bincount(cc, minlength=100)[50]


@pytest.mark.parametrize("n", [1, 7, 1000, 250007])
def test_select_ranks_exact(n):
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    t = _mixed_table(n, seed=100 + n)
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    probs = [0.01, 0.05, 0.1, 0.25, 0.5, 0.75, 0.9, 0.95, 0.99, 3 * (1 / 10), 1.0]
    ranks, exp = [], []
    for c in names:
        vals, valid = S.column_values(t, c)
        srt = np.sort(vals[valid].astype(np.float64))
        rk = engine.quantile_ranks(len(srt), probs)
        ranks.append(rk)
        exp.append([srt[r - 1] if r else np.nan for r in rk])
    got = engine.select_ranks(fr, names, np.array(ranks))
    assert np.array_equal(got, np.array(exp), equal_nan=True)   # exact order statistics


@pytest.fixture(params=["lsd", "lsd-onesweep", "partition"])
def sort_algo(request, monkeypatch):
    """Every implementation of the exact mode / distinct / order-statistic path: the LSD radix sort with its default
    three-kernel passes, with the one-sweep passes (ANV_SORT_ONESWEEP=1, read per call), and the partition + count path."""
    from anovos_b200 import engine
    if request.param == "lsd-onesweep":
        monkeypatch.setenv("ANV_SORT_ONESWEEP", "1")
    else:
        monkeypatch.delenv("ANV_SORT_ONESWEEP", raising=False)
    old, engine.sort_algorithm = engine.sort_algorithm, request.param.split("-")[0]
    yield request.param
    engine.sort_algorithm = old


@pytest.mark.parametrize("n", [1, 40, 5000, 200001])
def test_mode_distinct_exact(n, sort_algo):
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    rng = np.random.default_rng(n)
    t = _mixed_table(n, seed=200 + n)
    t = t.append_column("i32_small", pa.array(rng.integers(0, 7, n).astype(np.int32), mask=rng.random(n) < 0.2))
    t = t.append_column("f32_signed", pa.array(np.round(rng.normal(0, 3, n)).astype(np.float32)))
    # exact zeros are counted by the pack kernel and spliced back in: all-zero, zeros + nulls, -0.0, zero-inflated with
    # negatives on the left and a tie between the zero run and another value
    t = t.append_column("all_zero", pa.array(np.zeros(n, np.float32)))
    t = t.append_column("zero_or_null", pa.array(np.zeros(n, np.int64), mask=rng.random(n) < 0.5))
    zi = np.where(rng.random(n) < 0.6, 0.0, np.round(rng.normal(0, 50, n), 1))
    zi[rng.random(n) < 0.1] = -0.0
    t = t.append_column("f64_zero_inflated", pa.array(zi, mask=rng.random(n) < 0.05))
    tie = np.concatenate([np.zeros(n // 3), np.full(n // 3, -2.5), np.arange(n - 2 * (n // 3)) + 1.0])
    t = t.append_column("f32_zero_tie", pa.array(rng.permutation(tie).astype(np.float32)))
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    probs = [0.01, 0.25, 0.4, 0.5, 0.6, 0.75, 0.99, 1.0]
    rk = []
    for c in names:
        vals, valid = S.column_values(t, c)
        rk.append(engine.quantile_ranks(int(valid.sum()), probs))
    got, qv = engine.sort_mode_distinct(fr, names, np.array(rk))
    for i, c in enumerate(names):   # order statistics read from the sorted keys
        vals, valid = S.column_values(t, c)
        srt = np.sort(vals[valid].astype(np.float64))
        exp = [srt[r - 1] if r else np.nan for r in rk[i]]
        assert np.array_equal(qv[i], np.array(exp), equal_nan=True), c
    assert got == engine.sort_mode_distinct(fr, names)
    for c, (mode, rows, nd) in zip(names, got):
        vals, valid = S.column_values(t, c)
        x = vals[valid]
        if x.size == 0:
            assert (mode, rows, nd) == (None, None, 0)
            continue
        if x.dtype.kind == "f":
            x = x + 0.0
        u, k = np.unique(x, return_counts=True)
        assert nd == u.size, c                          # exact distinct
        assert rows == int(k.max()), c                  # exact mode_rows
        assert mode == u[np.argmax(k)].item(), c        # smallest value among ties; an int64 mode compares exactly


def test_hll_matches_oracle_registers(income):
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    fr = ColumnFrame.from_arrow(income)
    names = [c for c in income.column_names]
    for p in (9, 12):
        est = engine.hll_estimates(fr, names, p)
        for c, (e, band) in zip(names, est):
            vals, valid = S.column_values(income, c)
            sd = S.spark_dtype(income.schema.field(c).type)
            regs = S.hll_registers(S.hll_hashes(vals[valid], sd), p)
            assert (e, band) == S.hll_estimate(regs, p), (c, p)
    rng = np.random.default_rng(5)
    n = 300000
    t = pa.table({"f32": pa.array(rng.normal(0, 1, n).astype(np.float32), mask=rng.random(n) < 0.1),
                  "f64": pa.array(np.round(rng.normal(0, 100, n), 1)),
                  "i64": pa.array(rng.integers(-10**9, 10**9, n).astype(np.int64))})
    fr = ColumnFrame.from_arrow(t)
    for c, (e, band) in zip(t.column_names, engine.hll_estimates(fr, t.column_names, 14)):
        vals, valid = S.column_values(t, c)
        regs = S.hll_registers(S.hll_hashes(vals[valid], S.spark_dtype(t.schema.field(c).type)), 14)
        assert (e, band) == S.hll_estimate(regs, 14), c


def test_moments_hist_without_early_pivot():
    """Tiles whose first 1024+ rows are null / non-finite: the pivot fallback (null lanes
    impersonate 0) must not pollute min / max / nonzero counts / histograms."""
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    n = 70001
    rng = np.random.default_rng(11)
    a = (rng.normal(7.0, 1.0, n)).astype(np.float32)          # all values > 0: a stray 0 would show in min
    ma = np.zeros(n, bool); ma[:5000] = True; ma[rng.random(n) < 0.2] = True
    b = np.full(n, np.inf, np.float32); mb = rng.random(n) < 0.5   # only +inf values and nulls
    c = (-np.abs(rng.normal(3.0, 1.0, n))).astype(np.float32)  # all negative: a stray 0 would show in max
    mc = np.zeros(n, bool); mc[:40000] = True
    d = rng.integers(5, 50, n).astype(np.int32); md = np.zeros(n, bool); md[:3000] = True
    t = pa.table({"a": pa.array(a, mask=ma), "b": pa.array(b, mask=mb), "c": pa.array(c, mask=mc), "d": pa.array(d, mask=md)})
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    m = engine.moments(fr, names)
    for i, nme in enumerate(names):
        vals, valid = S.column_values(t, nme)
        x = vals[valid].astype(np.float64)
        assert m["n_valid"][i] == x.size and m["n_nonzero"][i] == np.count_nonzero(x != 0), nme
        assert m["min"][i] == x.min() and m["max"][i] == x.max(), nme
    cuts = [S.equal_range_cutoffs(float(m["min"][i]), float(m["max"][i]), 10) if np.isfinite(m["min"][i] - m["max"][i])
            else [1.0 * j for j in range(1, 10)] for i in range(len(names))]
    model = engine.BinModel(fr, names, cuts, [(float(m["min"][i]), float(m["max"][i])) for i in range(len(names))])
    h = engine.histogram(fr, model)
    m2, h2 = engine.moments_histogram(fr, model)
    assert (h == h2).all()
    for i, nme in enumerate(names):
        vals, valid = S.column_values(t, nme)
        exp = S.assign_bins(vals, valid, cuts[i], 10)
        assert np.array_equal(h[i, :11], np.bincount(exp, minlength=11).astype(np.uint64)), nme
        assert m2["min"][i] == m["min"][i] and m2["max"][i] == m["max"][i] and m2["n_nonzero"][i] == m["n_nonzero"][i]


@pytest.mark.parametrize("n", [300_007, 3_000_001])
def test_partition_count_adversarial_columns(n, monkeypatch):
    """The partition + count path on the inputs that stress it: heavy hitters below and above the splitter threshold,
    discrete columns (every key equals a splitter), a constant column, an all-null column, NaN runs, keys on both sides of
    zero, near-constant columns with a few outliers, sorted input (the sample positions are stratified) - against NumPy,
    and cell for cell against the LSD sort."""
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    rng = np.random.default_rng(n)
    heavy = rng.normal(0, 1, n).astype(np.float32)
    heavy[rng.random(n) < 0.2] = 1.25                      # 20 % one value
    heavy[rng.random(n) < 0.0003] = -7.5                   # ~ 1/P of the rows: may or may not become a splitter
    nanny = rng.normal(5, 2, n).astype(np.float32)
    nanny[rng.random(n) < 0.1] = np.nan
    spike = np.full(n, 3.0, np.float32)
    spike[rng.integers(0, n, 50)] = rng.normal(0, 1e6, 50).astype(np.float32)
    cols = {
        "normal": pa.array(rng.normal(27, 9, n).astype(np.float32)),
        "heavy": pa.array(heavy, mask=rng.random(n) < 0.01),
        "ints_small": pa.array(rng.integers(-3, 4, n).astype(np.int32)),
        "ints_wide": pa.array(rng.integers(-2 ** 31, 2 ** 31 - 1, n).astype(np.int32), mask=rng.random(n) < 0.3),
        "constant": pa.array(np.full(n, -4.5, np.float32)),
        "all_null": pa.array(np.zeros(n, np.float32), mask=np.ones(n, bool)),
        "nan_runs": pa.array(nanny),
        "spike": pa.array(spike),
        "sorted": pa.array(np.sort(rng.exponential(3, n)).astype(np.float32)),
        "zero_inflated": pa.array(np.where(rng.random(n) < 0.7, 0.0, rng.exponential(2, n)).astype(np.float32), mask=rng.random(n) < 0.3),
        "lognormal": pa.array(np.exp(rng.normal(0, 0.75, n)).astype(np.float32)),
    }
    t = pa.table(cols)
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    probs = [0.0001, 0.01, 0.05, 0.1, 0.25, 0.5, 0.75, 0.9, 0.95, 0.99, 1.0]
    rk = np.array([engine.quantile_ranks(n - t.column(c).null_count, probs) for c in names])
    old = engine.sort_algorithm
    try:
        engine.sort_algorithm = "partition"
        got, qv = engine.sort_mode_distinct(fr, names, rk)
        engine.sort_algorithm = "lsd"
        ref, qr = engine.sort_mode_distinct(fr, names, rk)
        monkeypatch.setenv("ANV_SORT_ONESWEEP", "1")           # the one-sweep passes give the same sorted keys
        one, q1 = engine.sort_mode_distinct(fr, names, rk)
        monkeypatch.delenv("ANV_SORT_ONESWEEP")
    finally:
        engine.sort_algorithm = old
    assert np.array_equal(q1, qr, equal_nan=True)
    def same(a, b):      # (mode, rows, distinct) tuples; the mode of a NaN-dominated column is NaN on both sides
        return a == b or (a[1:] == b[1:] and a[0] != a[0] and b[0] != b[0])
    assert all(same(a, b) for a, b in zip(got, ref)), [(n, a, b) for n, a, b in zip(names, got, ref) if not same(a, b)]
    assert all(same(a, b) for a, b in zip(one, ref))
    assert np.array_equal(qv, qr, equal_nan=True)
    for i, c in enumerate(names):
        vals, valid = S.column_values(t, c)
        x = vals[valid]
        if x.size == 0:
            assert got[i] == (None, None, 0)
            continue
        srt = np.sort(x.astype(np.float64))              # NaN last, like Spark
        exp = [srt[r - 1] if r else np.nan for r in rk[i]]
        assert np.array_equal(qv[i], np.array(exp), equal_nan=True), c
        if x.dtype.kind == "f":
            x = x + 0.0
        u, k = np.unique(x, return_counts=True)          # equal_nan: all NaNs are one value
        assert got[i][2] == u.size and got[i][1] == int(k.max()), c
        best = u[k == k.max()]
        assert got[i][0] == float(np.nanmin(best)) or (np.isnan(got[i][0]) and np.isnan(best).all()), c


@pytest.mark.parametrize("n", [1, 777, 250_003])
def test_hll_registers_from_the_sorted_runs_equal_the_hll_kernel(n):
    """anv_mode_distinct_hll: the registers hashed from one key per run of the sorted keys (+ the zero run) are the
    registers anv_hll_registers computes from every value - all dtypes, nulls, zeros, -0.0, NaN, 32- and 64-bit key groups."""
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    rng = np.random.default_rng(n)
    f = rng.normal(0, 3, n).astype(np.float32)
    f[rng.random(n) < 0.2] = 0.0
    f[rng.random(n) < 0.05] = -0.0
    f[rng.random(n) < 0.03] = np.nan
    d = np.round(rng.normal(-1e6, 250, n), 1)
    d[rng.random(n) < 0.02] = np.nan
    t = pa.table({"f32": pa.array(f, mask=rng.random(n) < 0.1), "i32": pa.array(rng.integers(-5, 6, n).astype(np.int32)),
                  "f64": pa.array(d, mask=rng.random(n) < 0.3), "i64": pa.array(rng.integers(-2 ** 40, 2 ** 40, n)),
                  "all_null": pa.array(np.zeros(n, np.float32), mask=np.ones(n, bool)),
                  "wide": pa.array(rng.normal(0, 1e3, n).astype(np.float32))})
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    for p in (9, 12):
        res, _, regs = engine.sort_mode_distinct(fr, names, None, hll_p=p)
        assert res == engine.sort_mode_distinct(fr, names) or all(a[1:] == b[1:] for a, b in zip(res, engine.sort_mode_distinct(fr, names)))
        assert np.array_equal(regs, engine.hll_registers(fr, names, p)), p


@pytest.mark.parametrize("n", [1, 1000, 2048 * 4 + 5, 300_001, 2_500_003])
def test_fused_pass_staged_equals_register_staged(n, monkeypatch):
    """The cp.async-staged fused moments + histogram kernel (default) against the register-staged one (ANV_FUSED_STAGED=0,
    read per call): same vector -> thread mapping, so moments and counts are equal BIT FOR BIT; both equal the separate
    moments and histogram kernels.  Sizes cover: no full group, drain only, steady state + drain, several tiles."""
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    t = _mixed_table(n, seed=n % 97, null_rate=0.15).drop_columns(["f32_allnull"])
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    mom = engine.moments(fr, names)
    cuts, lohi = [], []
    for i, c in enumerate(names):
        mn, mx = float(mom["min"][i]), float(mom["max"][i])
        cuts.append(S.equal_range_cutoffs(mn, mx, 10))
        lohi.append((mn, mx))
    model = engine.BinModel(fr, names, cuts, lohi)
    h = engine.histogram(fr, model)
    out = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("ANV_FUSED_STAGED", flag)
        out[flag] = engine.moments_histogram(fr, model)
    (m0, h0), (m1, h1) = out["0"], out["1"]
    assert (h0 == h1).all() and (h0 == h).all()
    for f in engine.MOMENT_FIELDS:
        assert np.array_equal(m0[f], m1[f], equal_nan=True), f
        assert np.array_equal(mom[f], m1[f], equal_nan=True), f
