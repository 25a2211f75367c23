"""The per-value rules of invalidEntries_detection (reference data_analyzer/quality_checker.py:1504-1607) and the tables
the membership pass (csrc/invalid.cu) searches.

Every verdict is a pure function of one value, so the host decides once which distinct values are invalid and the GPU
pass counts and nulls the rows holding them:
  - string columns: the rule runs once per dictionary entry -> a table of dictionary codes;
  - int / bigint columns in "auto" mode: the closed-form set of AUTO_INT_VALUES, no data-dependent step;
  - every other numeric case: the rule runs over the column's distinct values (str(int(x)) or str(float(x)), what the
    reference's Python UDF sees).
Tables are sorted ascending in numeric order (-0.0 before 0.0, NaN last) with one entry per distinct value."""
from __future__ import annotations

import re

import numpy as np

NULL_VOCAB = ["", " ", "nan", "null", "na", "inf", "n/a", "not defined", "none", "undefined", "blank", "unknown"]
SPECIAL_CHARS_VOCAB = ["&", "$", ";", ":", ".", ",", "*", "#", "@", "_", "?", "%", "!", "^", "(", ")", "-", "/", "'"]
_VOCAB = frozenset(NULL_VOCAB + SPECIAL_CHARS_VOCAB)
_REPEAT = re.compile(r"\b([a-zA-Z0-9])\1\1+\b")

DETECTION_TYPES = ("auto", "manual", "both")


def auto_invalid(e: str) -> bool:
    """The auto rules on e = str(v).lower().strip(): a null / special-character token, a run of three or more identical
    alphanumerics between word boundaries, or three or more code points each one above the previous."""
    if e in _VOCAB or _REPEAT.search(e):
        return True
    return len(e) >= 3 and all(ord(e[i]) - ord(e[i - 1]) == 1 for i in range(1, len(e)))


class Rule:
    """One column's verdict on a value's string form.  Unlike the reference's UDF (which, in "manual" / "both" mode,
    can append two flags for one value and so shift every later column's flags), each value gets exactly one verdict:
    invalid when any invalid_entries pattern matches it or, with valid_entries given, none of those matches it."""

    def __init__(self, detection_type="auto", invalid_entries=(), valid_entries=(), partial_match=False):
        self.auto = detection_type in ("auto", "both")
        self.manual = detection_type in ("manual", "both")
        self.invalid = [re.compile(r) for r in invalid_entries]
        self.valid = [re.compile(r) for r in valid_entries]
        self.partial = bool(partial_match)

    def _matches(self, p, e):
        return (p.search(e) if self.partial else p.fullmatch(e)) is not None

    def __call__(self, s: str) -> bool:
        e = s.lower().strip()
        if self.auto and auto_invalid(e):
            return True
        if self.manual:
            if any(self._matches(p, e) for p in self.invalid):
                return True
            if self.valid and not any(self._matches(p, e) for p in self.valid):
                return True
        return False

    @property
    def auto_only(self):
        return self.auto and not self.manual

    @property
    def flags_nothing(self):
        return not self.auto and not self.manual


def _auto_ints():
    vals = set()
    for n in range(3, 20):
        for d in "123456789":
            vals.add(int(d * n))
            vals.add(-int(d * n))
    for n in range(3, 10):
        for s in range(1, 11 - n):
            vals.add(int("".join(str(s + i) for i in range(n))))
    return sorted(v for v in vals if -(1 << 63) <= v < (1 << 63))


# Python int strings the auto rules flag: repdigits of 3+ digits of either sign (111, -999, ...) and positive runs of
# 3+ ascending consecutive digits (123 ... 123456789).  156 of them fit in int32, 332 in int64.
AUTO_INT_VALUES = _auto_ints()
AUTO_INT64 = np.array(AUTO_INT_VALUES, np.int64)
AUTO_INT32 = AUTO_INT64[(AUTO_INT64 >= -(1 << 31)) & (AUTO_INT64 < (1 << 31))].astype(np.int32)

_CANON_NAN = {np.dtype(np.float32): np.uint32(0x7FC00000), np.dtype(np.float64): np.uint64(0x7FF8000000000000)}


def canonical_nan_bits(values: np.ndarray) -> np.ndarray:
    """float array -> the same values with every NaN payload replaced by the one quiet NaN the kernel compares with."""
    values = np.asarray(values)
    if values.dtype.kind != "f":
        return values
    bits = values.view(np.uint32 if values.itemsize == 4 else np.uint64).copy()
    bits[np.isnan(values)] = _CANON_NAN[values.dtype]
    return bits.view(values.dtype)


def ordered_keys(values: np.ndarray) -> np.ndarray:
    """int32 / int64 / float32 / float64 values -> the unsigned keys whose order is numeric order (the kernel's key
    transform): signed integers flip the sign bit; floats flip every bit when negative and the sign bit otherwise, so
    -0.0 < 0.0 and NaN (canonicalised first) sorts above +inf."""
    values = canonical_nan_bits(np.asarray(values))
    u = np.uint32 if values.itemsize == 4 else np.uint64
    bits = values.view(u)
    top = u(1 << (8 * values.itemsize - 1))
    if values.dtype.kind in "iu":
        return bits ^ top
    neg = (bits & top) != 0
    return np.where(neg, ~bits, bits | top).astype(u)


def sort_table(values: np.ndarray) -> np.ndarray:
    """Distinct values in key order (what engine.flag_members takes)."""
    values = canonical_nan_bits(np.asarray(values))
    keys = ordered_keys(values)
    _, first = np.unique(keys, return_index=True)
    return values[first]


def value_str(v, is_float: bool) -> str:
    """What the reference's UDF and its `str(x)` of collected values show: Python's str of an int or a float."""
    return str(float(v)) if is_float else str(int(v))


def numeric_table(distinct: np.ndarray, rule: Rule) -> np.ndarray:
    """Distinct values of a numeric column (any order, NaN payloads canonical or not) -> the invalid ones, in key order."""
    distinct = sort_table(distinct)
    is_float = distinct.dtype.kind == "f"
    keep = np.fromiter((rule(value_str(v, is_float)) for v in distinct.tolist()), bool, len(distinct))
    return distinct[keep]


def int_auto_table(dtype) -> np.ndarray:
    return AUTO_INT32 if np.dtype(dtype) == np.int32 else AUTO_INT64


def dictionary_table(dictionary, rule: Rule) -> np.ndarray:
    """Dictionary entries -> the int32 codes of the invalid ones, ascending (a null entry is never invalid)."""
    return np.array([i for i, s in enumerate(dictionary) if s is not None and rule(str(s))], np.int32)
