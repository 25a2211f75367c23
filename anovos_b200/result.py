"""Result object of the GPU path: the small per-attribute frames the reference returns as
Spark DataFrames.  Callers of the reference immediately do `.toPandas().to_csv(...)`
(data_report/report_preprocessing.py:92), `.show(n)` (workflow.py:509), `.count()` or
`.where(F.col("attribute") == x)` (reference tests); this class offers that surface on top
of a pandas DataFrame."""
from __future__ import annotations

import numpy as np
import pandas as pd


def _column_array(v):
    """One result column -> what the pandas constructor would make of it (same dtype inference), without its overhead for
    the two common cases: a NumPy array (taken as is, copied) and a list of str."""
    if isinstance(v, np.ndarray):
        return v.copy()
    if isinstance(v, list) and v and all(type(x) is str for x in v):
        return pd.array(v, dtype="str")
    return pd.Series(v).array


def build_frame(columns: dict, attrs=None) -> pd.DataFrame:
    """pandas frame of equally long columns (dict name -> ndarray | list), RangeIndex; equal to pd.DataFrame(columns)."""
    names = list(columns)
    n = len(columns[names[0]]) if names else 0
    try:
        if n == 0:
            raise TypeError("empty result: let the pandas constructor infer the dtypes")
        df = pd.DataFrame._from_arrays([_column_array(columns[k]) for k in names], columns=pd.Index(names), index=pd.RangeIndex(n),
                                       verify_integrity=False)
    except (AttributeError, TypeError):          # a pandas without the fast constructor
        df = pd.DataFrame({k: columns[k] for k in names})
    if attrs:
        df.attrs.update(attrs)
    return df


class ResultFrame:
    def __init__(self, df: pd.DataFrame):
        self._columns = self._attrs = None
        idx = df.index
        plain = isinstance(idx, pd.RangeIndex) and idx.start == 0 and idx.step == 1
        self._frame = df if plain else df.reset_index(drop=True)

    @classmethod
    def from_columns(cls, columns: dict, attrs=None) -> "ResultFrame":
        """Result of per-attribute columns (name -> ndarray | list): the pandas frame is built when it is asked for, a
        fresh one per toPandas() call (no defensive copy of a stored frame)."""
        self = cls.__new__(cls)
        self._columns, self._attrs, self._frame = dict(columns), attrs, None
        return self

    @property
    def _df(self) -> pd.DataFrame:
        if self._frame is None:
            self._frame = build_frame(self._columns, self._attrs)
        return self._frame

    def toPandas(self) -> pd.DataFrame:
        if self._columns is not None:
            return build_frame(self._columns, self._attrs)
        return self._frame.copy()

    to_pandas = toPandas

    @property
    def columns(self):
        return list(self._columns) if self._columns is not None else list(self._df.columns)

    def count(self) -> int:
        return len(self._df)

    def show(self, n: int = 20, truncate=True):
        with pd.option_context("display.max_columns", None, "display.width", 200):
            print(self._df.head(n).to_string(index=False))

    def where(self, cond) -> "ResultFrame":
        """cond: pandas query string ("attribute == 'age'"), a callable df -> mask, or a
        dict {column: value}."""
        if isinstance(cond, str):
            return ResultFrame(self._df.query(cond))
        if isinstance(cond, dict):
            m = pd.Series(True, index=self._df.index)
            for k, v in cond.items():
                m &= self._df[k] == v
            return ResultFrame(self._df[m])
        return ResultFrame(self._df[cond(self._df)])

    filter = where

    def select(self, *cols) -> "ResultFrame":
        cols = list(cols[0]) if len(cols) == 1 and isinstance(cols[0], (list, tuple)) else list(cols)
        return ResultFrame(self._df[cols])

    def collect(self):
        return [tuple(r) for r in self._df.itertuples(index=False)]

    def to_csv(self, path, **kw):
        kw.setdefault("index", False)
        return self._df.to_csv(path, **kw)

    def __len__(self):
        return len(self._df)

    def __repr__(self):
        return "ResultFrame(%d rows x %d cols: %s)" % (len(self._df), self._df.shape[1], ", ".join(self.columns))
