"""GPU tests of the binning kernels at every bin count where their counting path or threshold table changes, up to the
ANV_MAX_BINS = 16 384 limit, against exact references.

`hist_smem` picks the counting path from count_stride = B + 1: private per-thread counters up to B = 39 (moments and
histogram fused in one kernel), per-CTA shared uint32 counters up to B = 10 239, global 64-bit atomics up to B = 16 384.
The threshold table holds the next power of two of B slots plus two, 8 bytes each, in shared memory: the launch opts in
to more than 40 KB from B = 2 049 (histograms) and B = 4 097 (bin ids), and needs 131 KB at B = 16 384.

* kernels: the adversarial columns of test_gpu_kernel_edges (every native threshold and one step either side, the
  cutoffs, lo / hi and one step outside, NaN, +-inf, +-0.0, subnormals, the integer extremes, 20 % of rows over three times
  the model's range, 5 % nulls) in f32 / f64 / i32 / i64, binned by the equal_range guess and by the binary search, on
  each side of every switch - against `oracle.exact.exact_bins` + np.bincount, resident and in row chunks;
* API: attribute_binning, drift_detector.statistics and IV / IG_calculation with thousands of bins - against the oracle.
Every input is built from a seed."""
import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu

import test_gpu_kernel_edges as E
from oracle import api as O
from oracle import exact as X
from oracle import spark_semantics as S

# each side of the path 0 / 1 switch, every threshold-table doubling (2 049: the > 40 KB opt-in of the histograms, 4 097:
# of the bin ids), the path 1 / 2 switch and the maximum
WIDE_B = [39, 40, 41, 2048, 2049, 4096, 4097, 8192, 8193, 10239, 10240, 16383, 16384]
N_ROWS = 200_003      # odd: ragged vectors and a scalar tail; a dozen 16 384-row tiles per column
CHUNK = 70_016        # row chunks: a multiple of 32 (the bitmap words) but not of any tile size


def _expected(t, names, cuts):
    return [X.exact_bins(*E._col_values(t, c), cuts[i]) for i, c in enumerate(names)]


def _check_bins(fr, model, names, exp, label, monkeypatch):
    """Histograms (anv_hist, anv_moments_hist with either staging) and bin ids (anv_bin_assign) of `model` on `fr` equal
    the reference ids `exp` and their bincounts, slot for slot over the whole count stride.  -> {staging flag: moments}."""
    from anovos_b200 import engine
    stride = model.max_bins + 1
    got, moms = {"histogram": engine.histogram(fr, model)}, {}
    for flag in ("0", "1"):
        monkeypatch.setenv("ANV_FUSED_STAGED", flag)
        moms[flag], got["moments_histogram staged=" + flag] = engine.moments_histogram(fr, model)
    monkeypatch.delenv("ANV_FUSED_STAGED")
    ids = engine.bin_assign(fr, model).cpu().numpy()
    assert ids.shape == (len(names), fr.n_rows), label
    for i, c in enumerate(names):
        bad = np.flatnonzero(ids[i] != exp[i])
        assert bad.size == 0, (label, c, bad.size, [(int(j), int(ids[i][j]), int(exp[i][j])) for j in bad[:5]])
        want = np.bincount(exp[i], minlength=stride).astype(np.uint64)
        for k, h in got.items():
            assert h.shape == (len(names), stride), (label, k)
            diff = np.flatnonzero(h[i] != want)
            assert diff.size == 0, (label, c, k, [(int(s), int(h[i][s]), int(want[s])) for s in diff[:5]])
    return moms


def _check_chunked(fr, model, names, exp, label):
    """The same model over row chunks: the summed histograms and the concatenated bin ids of the chunks."""
    from anovos_b200 import engine
    from anovos_b200.partitioned import PartitionedFrame
    pf = PartitionedFrame.from_frame(fr, CHUNK)
    assert pf.n_chunks > 2
    want = np.stack([np.bincount(e, minlength=model.max_bins + 1) for e in exp]).astype(np.uint64)
    assert np.array_equal(engine.histogram(pf, model), want), label
    assert np.array_equal(engine.moments_histogram(pf, model)[1], want), label
    ids = np.concatenate([engine.bin_assign(ch, model).cpu().numpy() for ch in pf.chunks(names)], axis=1)
    assert np.array_equal(ids, np.stack(exp)), label


def _wide_models(B, n):
    """test_gpu_kernel_edges' models at B bins, plus null-free copies of two columns: without a bitmap the fused kernel
    (B = 39) runs its cp.async-staged loop when ANV_FUSED_STAGED=1."""
    rng = np.random.default_rng(20_000 + B)
    cols, cuts, lohi, expect_mode = E._binning_models(B, rng, n)
    for c in ("f32_r0", "f64_r1"):
        i = list(cols).index(c)
        cols[c + "_dense"] = (cols[c][0], None)
        cuts.append(cuts[i])
        lohi.append(lohi[i])
        expect_mode.append(expect_mode[i])
    return cols, cuts, lohi, expect_mode


@pytest.mark.parametrize("B", WIDE_B)
def test_wide_bins_on_and_around_every_threshold(B, monkeypatch):
    from anovos_b200 import engine
    cols, cuts, lohi, expect_mode = _wide_models(B, N_ROWS)
    t, fr = E._frame(cols)
    names = t.column_names
    model = engine.BinModel(fr, names, cuts, lohi)
    assert model.max_bins == B
    for i, c in enumerate(names):                       # the guess where the model has lo / hi, the search elsewhere
        assert model.specs_host["mode"][i] == expect_mode[i], (c, B)
    exp = _expected(t, names, cuts)
    moms = _check_bins(fr, model, names, exp, B, monkeypatch)
    if B >= 40:
        # the unfused moments_histogram runs the K1 kernel of anv_moments, then the histogram kernel: same moments, bit
        # for bit (NaN payloads included)
        ref = engine.moments(fr, names)
        for flag, m in moms.items():
            assert m.tobytes() == ref.tobytes(), (B, flag)
    if B in (39, 4097, 10240, 16384):                   # one per counting path and the bin-id opt-in
        _check_chunked(fr, model, names, exp, B)


def test_mixed_bin_counts_in_one_launch(monkeypatch):
    """Columns of 3, 41 and 12 000 bins in one call: the count stride, and so the counting path (global atomics), comes
    from the widest column, while each column sizes its own threshold table from its own n_bins (a search over 4, 64 and
    16 384 slots).
    f32 columns take the guess, the others the search."""
    from anovos_b200 import engine
    rng = np.random.default_rng(12_000)
    cols, cuts, lohi = {}, [], []
    for dt, (lo, hi) in (("f32", (0.0, 1.0)), ("f64", (-1.0, 1.0)), ("i32", (-5000.0, 5000.0)), ("i64", (-1e12, 1e12))):
        for B in (3, 41, 12_000):
            cut = S.equal_range_cutoffs(lo, hi, B)
            cols["%s_b%d" % (dt, B)] = E._tile(E._catalogue(dt, cut, lo, hi), N_ROWS, rng, lo, hi, dt)
            cuts.append(cut)
            lohi.append((lo, hi) if dt == "f32" else None)
    t, fr = E._frame(cols)
    names = t.column_names
    model = engine.BinModel(fr, names, cuts, lohi)
    assert model.max_bins == 12_000
    assert [int(m) for m in model.specs_host["mode"]] == [1, 1, 1] + [0] * 9
    exp = _expected(t, names, cuts)
    _check_bins(fr, model, names, exp, "mixed", monkeypatch)
    _check_chunked(fr, model, names, exp, "mixed")


def test_duplicate_and_nan_cutoffs_at_5000_bins(monkeypatch):
    """Equal-frequency cutoffs of 5 000 bins on zero-inflated columns and on columns of about 50 distinct values: runs of
    thousands of equal thresholds for the binary search.  Copies of the 50-value columns get NaN cutoffs in front, which
    native_thresholds maps to the type's lowest value: a NaN cutoff is below every value (`v <= NaN` is False)."""
    from anovos_b200 import engine
    rng = np.random.default_rng(5000)
    n = N_ROWS
    zero = np.where(rng.random(n) < 0.8, 0.0, rng.exponential(3.0, n))
    few = rng.integers(0, 50, n)
    base = {"f32_zero": zero.astype(np.float32), "f64_zero": zero, "i32_zero": (zero * 100).astype(np.int32),
            "f32_few": (few * 0.25 - 3).astype(np.float32), "f64_few": few / 3.0 - 1e6,
            "i32_few": (few * 7 - 100).astype(np.int32), "i64_few": few.astype(np.int64) * 2 ** 40 - 2 ** 45}
    cols, cuts = {}, []
    for k, v in base.items():
        m = rng.random(n) < 0.05
        cut = S.equal_frequency_cutoffs(np.sort(v[~m].astype(np.float64)), 5000)
        assert len(cut) - len(set(cut)) > 3500          # thousands of equal thresholds
        cols[k] = (v, m)
        cuts.append(cut)
        if k.endswith("_few"):
            cols[k + "_nan_cuts"] = (v, m)
            cuts.append([float("nan")] * 300 + cut[300:])
    t, fr = E._frame(cols)
    names = t.column_names
    model = engine.BinModel(fr, names, cuts, None)
    assert model.max_bins == 5000
    # the reference has no NaN cutoffs: below every value of these columns is -inf
    exp = _expected(t, names, [[-np.inf if c != c else c for c in cut] for cut in cuts])
    for i, c in enumerate(names):
        if c.endswith("_nan_cuts"):
            assert exp[i][exp[i] > 0].min() > 300, c    # no value lands in the bins below the NaN cutoffs
    _check_bins(fr, model, names, exp, "duplicates", monkeypatch)


# ---- the API against the oracle ---------------------------------------------------------------------------------------

PLAIN = ["f32", "f64", "i32", "i64"]                    # nulls only: equal_range takes min / max over them
SPECIAL = ["f32_inf_nan", "f64_inf_nan"]                 # + NaN and +-inf: equal_frequency only


def _api_table(seed, shift=0.0):
    """~200 k rows of all four numeric dtypes with 5 % nulls, and two float columns with +-inf on 1 % of the rows each
    and five NaNs: fewer NaNs than one bin of 16 384 holds, so no equal-frequency cutoff is NaN.  Plus a 0 / 1 label."""
    rng = np.random.default_rng(seed)
    n = N_ROWS

    def nulls():
        return rng.random(n) < 0.05

    def special(x):
        u = rng.random(n)
        x = np.where(u < 0.01, -np.inf, np.where(u > 0.99, np.inf, x)).astype(x.dtype)
        x[rng.choice(n, 5, replace=False)] = np.nan
        return x

    f32 = rng.normal(10.0 + shift, 3.0, n).astype(np.float32)
    f64 = rng.normal(-1e6 + 100 * shift, 250.0, n)
    return pa.table({
        "f32": pa.array(f32, mask=nulls()),
        "f64": pa.array(f64, mask=nulls()),
        "i32": pa.array(rng.integers(-30_000, 30_000 + int(3000 * shift), n).astype(np.int32), mask=nulls()),
        "i64": pa.array(rng.integers(-2 ** 40, 2 ** 40, n).astype(np.int64) + int(2 ** 36 * shift), mask=nulls()),
        "f32_inf_nan": pa.array(special(rng.lognormal(0.0, 1.0 + shift, n).astype(np.float32)), mask=nulls()),
        "f64_inf_nan": pa.array(special(rng.normal(0.0, 1e-3, n)), mask=nulls()),
        "label": pa.array((rng.random(n) < 1.0 / (1.0 + np.exp(-(f32 - 10.0) / 3.0))).astype(np.int32)),
    })


@pytest.fixture(scope="module")
def api_table():
    return _api_table(7)


def _ids(fr, c):
    """(bin ids, valid) of a binned column of a resident frame."""
    d, v = fr.column(c).device()
    ok = np.ones(fr.n_rows, bool) if v is None else \
        np.unpackbits(v.cpu().numpy().view(np.uint8), bitorder="little")[:fr.n_rows].astype(bool)
    return d.cpu().numpy(), ok


@pytest.mark.parametrize("bin_size", [41, 5000, 16384])
@pytest.mark.parametrize("method", ["equal_range", "equal_frequency"])
def test_attribute_binning_vs_oracle(api_table, method, bin_size):
    import anovos.data_transformer.transformers as tr
    from anovos_b200.partitioned import PartitionedFrame
    t = api_table
    cols = PLAIN if method == "equal_range" else PLAIN + SPECIAL
    exp = O.attribute_binning(t, list_of_cols=cols, method_type=method, bin_size=bin_size)
    got = tr.attribute_binning(None, t, list_of_cols=cols, method_type=method, bin_size=bin_size)
    chunked = tr.attribute_binning(None, PartitionedFrame.from_frame(t, CHUNK), list_of_cols=cols, method_type=method,
                                   bin_size=bin_size).materialize(cols)
    for c in cols:
        e = exp.column(c).combine_chunks()
        e_ids, e_ok = np.asarray(e.fill_null(0)), np.asarray(e.is_valid())
        if method == "equal_range":
            assert e_ids.max() == bin_size, c           # the maximum lands in the last bin
        for label, fr in (("resident", got), ("chunked", chunked)):
            ids, ok = _ids(fr, c)
            assert np.array_equal(ok, e_ok), (label, c)
            bad = np.flatnonzero(ids != e_ids)
            assert bad.size == 0, (label, method, bin_size, c, [(int(j), int(ids[j]), int(e_ids[j])) for j in bad[:5]])


def test_categorical_labels_with_5000_bins(api_table):
    import anovos.data_transformer.transformers as tr
    t = api_table
    got = tr.attribute_binning(None, t, list_of_cols=PLAIN, bin_size=5000, bin_dtype="categorical")
    exp = O.attribute_binning(t, list_of_cols=PLAIN, bin_size=5000, bin_dtype="categorical")
    for c in PLAIN:
        col = got.column(c)
        assert len(col.dictionary) == 5000, c
        codes, ok = _ids(got, c)
        labels = [col.dictionary[k] if v else None for k, v in zip(codes.tolist(), ok.tolist())]
        assert labels == exp.column(c).to_pylist(), c


@pytest.mark.parametrize("bin_method", ["equal_range", "equal_frequency"])
def test_drift_with_12000_bins_vs_oracle(bin_method, tmp_path):
    import anovos.drift_stability.drift_detector as dd
    src, tgt = _api_table(11), _api_table(12, shift=0.3)
    kw = dict(list_of_cols=PLAIN, method_type="all", bin_method=bin_method, bin_size=12_000, use_sampling=False)
    got = dd.statistics(None, tgt, src, source_path=str(tmp_path / "g"), **kw).toPandas()
    exp = O.statistics(tgt, src, source_path=str(tmp_path / "o"), **kw)
    assert got["attribute"].tolist() == exp["attribute"].tolist() == PLAIN
    for m in ("PSI", "HD", "JSD", "KS"):
        g, e = got[m].values.astype(float), np.array([0.0 if v is None else v for v in exp[m].tolist()], float)
        assert np.allclose(g, e, rtol=1e-9, atol=1e-12), (m, g, e)    # test_gpu_api.py::test_drift_vs_oracle's tolerance
    assert got["flagged"].tolist() == exp["flagged"].tolist()


@pytest.mark.parametrize("bin_method", ["equal_range", "equal_frequency"])
def test_iv_ig_with_5000_bins_vs_oracle(api_table, bin_method):
    import anovos.data_analyzer.association_evaluator as ae
    t = api_table
    cols = PLAIN if bin_method == "equal_range" else PLAIN + SPECIAL
    enc = {"bin_method": bin_method, "bin_size": 5000, "monotonicity_check": 0}
    for fn, key in (("IV_calculation", "iv"), ("IG_calculation", "ig")):
        got = getattr(ae, fn)(None, t, list_of_cols=cols, label_col="label", encoding_configs=enc).toPandas()
        exp = getattr(O, fn)(t, list_of_cols=cols, label_col="label", encoding_configs=enc)
        assert got["attribute"].tolist() == exp["attribute"].tolist() == cols
        # same counts; the per-group terms are summed in another order (all of one sign: <= 5 000 * 2^-53 relative)
        assert np.allclose(got[key].values.astype(float), exp[key].values.astype(float), rtol=1e-12, atol=1e-14), fn
