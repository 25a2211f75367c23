"""The 16 384-bin limit of the binning kernels (ANV_MAX_BINS) through the product's host layer, on the NumPy stand-in of
tests/cpu_engine.py: every entry point that takes a bin_size refuses one above the limit with a ValueError that names it,
before any device work; a binning model with more bins, such as a saved one, is refused too; the limit itself is
accepted."""
import warnings

import numpy as np
import pyarrow as pa
import pytest

import cpu_engine
from oracle import api as O

N = 5003


def _table():
    rng = np.random.default_rng(16384)
    return pa.table({"x": pa.array(rng.normal(0, 1, N).astype(np.float32), mask=rng.random(N) < 0.05),
                     "k": pa.array(rng.integers(-40000, 40000, N).astype(np.int64)),
                     "label": pa.array(rng.integers(0, 2, N).astype(np.int32))})


@pytest.fixture
def no_device():
    """The stand-in with every engine pass and the device check replaced by a failure."""
    from anovos_b200 import _lib, engine

    def device_work(*a, **k):
        raise AssertionError("device work before the bin_size check")
    with cpu_engine.installed(), pytest.MonkeyPatch.context() as mp:    # undone before the stand-in is removed
        mp.setattr(_lib, "require_cuda", device_work)
        for n in ("moments", "histogram", "moments_histogram", "bin_assign", "code_counts", "select_ranks",
                  "sort_mode_distinct", "class_hist"):
            mp.setattr(engine, n, device_work)
        yield


def test_bin_size_above_the_limit_is_refused_before_device_work(no_device, tmp_path):
    import anovos.data_analyzer.association_evaluator as ae
    import anovos.data_transformer.transformers as tr
    import anovos.drift_stability.drift_detector as dd
    from anovos_b200 import _lib
    t, big = _table(), _lib.MAX_BINS + 1
    calls = {
        "attribute_binning": lambda: tr.attribute_binning(None, t, list_of_cols=["x", "k"], bin_size=big),
        "attribute_binning equal_frequency": lambda: tr.attribute_binning(None, t, list_of_cols=["x"],
                                                                          method_type="equal_frequency", bin_size=big),
        "monotonic_binning": lambda: tr.monotonic_binning(None, t, list_of_cols=["x"], bin_size=big),
        "statistics": lambda: dd.statistics(None, t, t, list_of_cols=["x", "k"], bin_size=big, use_sampling=False,
                                            source_path=str(tmp_path)),
    }
    for fn in ("IV_calculation", "IG_calculation"):
        for m in (0, 1):
            enc = {"bin_method": "equal_range", "bin_size": big, "monotonicity_check": m}
            calls["%s monotonicity_check=%d" % (fn, m)] = \
                lambda fn=fn, enc=enc: getattr(ae, fn)(None, t, list_of_cols=["x", "k"], encoding_configs=enc)
    for name, call in calls.items():
        with pytest.raises(ValueError, match="bin_size 16385: at most 16384 bins"):
            call()
        assert not (tmp_path / "drift_statistics").exists(), name


def test_model_with_more_bins_than_the_limit_is_refused(tmp_path):
    import anovos.data_transformer.transformers as tr
    import anovos.drift_stability.drift_detector as dd
    from anovos_b200 import _lib, engine
    from anovos_b200.data_transformer.transformers import save_binning_model
    from anovos_b200.frame import ColumnFrame
    t = _table()
    wide = [float(v) for v in np.linspace(-3, 3, _lib.MAX_BINS)]          # MAX_BINS cutoffs: one bin too many
    fr = ColumnFrame.from_arrow(t)
    with pytest.raises(ValueError, match="16385 bins .*'x'.* at most 16384"):
        engine.BinModel(fr, ["k", "x"], [[0.0], wide], None)
    save_binning_model(str(tmp_path / "ab"), ["x"], [wide])
    save_binning_model(str(tmp_path / "dd" / "drift_statistics"), ["x"], [wide])
    with cpu_engine.installed():
        with pytest.raises(ValueError, match="at most 16384 bins"):
            tr.attribute_binning(None, t, list_of_cols=["x"], pre_existing_model=True, model_path=str(tmp_path / "ab"))
        with pytest.raises(ValueError, match="at most 16384 bins"):
            dd.statistics(None, t, None, list_of_cols=["x"], pre_existing_source=True, use_sampling=False,
                          source_path=str(tmp_path / "dd"))


def test_bin_size_at_the_limit_is_accepted():
    import anovos.data_transformer.transformers as tr
    from anovos_b200 import _lib
    t = _table()
    with cpu_engine.installed(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = tr.attribute_binning(None, t, list_of_cols=["x", "k"], bin_size=_lib.MAX_BINS)
        ids = {c: got.column(c).device()[0].numpy() for c in ("x", "k")}
    exp = O.attribute_binning(t, list_of_cols=["x", "k"], bin_size=_lib.MAX_BINS)
    for c in ("x", "k"):
        e = np.asarray(exp.column(c).combine_chunks().fill_null(0))
        assert np.array_equal(ids[c], e) and e.max() == _lib.MAX_BINS, c
