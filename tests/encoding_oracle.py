"""A pure-Python restatement of the reference's categorical encoders on pyarrow tables (the oracle of
tests/test_encoding_cpu.py and tests/test_gpu_encoding.py): cat_to_num_unsupervised, cat_to_num_supervised and
outlier_categories (reference data_transformer/transformers.py:506-962, 3489-3671) with Spark 3's StringIndexer /
OneHotEncoder / pivot / window semantics, row by row, without the product's code counts or kernels.

Columns come in first-seen list order (where the reference iterates a set), strings compare in UTF-8 byte order, a
coverage cut among tied categories keeps the UTF-8 first, and the supervised model_path="NA" round trip is skipped - the
product's documented choices."""
from collections import Counter
from decimal import ROUND_HALF_UP, Decimal

import pyarrow as pa


def _u(s):
    return s.encode("utf-8")


def _cols(table, list_of_cols, drop_cols, extra_drop=()):
    cat = [f.name for f in table.schema if pa.types.is_string(f.type) or pa.types.is_large_string(f.type)]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = cat
    if isinstance(list_of_cols, str):
        list_of_cols = [x.strip() for x in list_of_cols.split("|")]
    if isinstance(drop_cols, str):
        drop_cols = [x.strip() for x in drop_cols.split("|")]
    return cat, list(list_of_cols), list(drop_cols) + list(extra_drop)


def round4(x):
    """F.round(x, 4): HALF_UP on the shortest repr."""
    return float(Decimal(repr(x)).quantize(Decimal("0.0001"), rounding=ROUND_HALF_UP))


def indexer_labels(values, index_order):
    cnt = Counter(v for v in values if v is not None)
    if index_order == "frequencyDesc":
        return sorted(cnt, key=lambda k: (-cnt[k], _u(k)))
    if index_order == "frequencyAsc":
        return sorted(cnt, key=lambda k: (cnt[k], _u(k)))
    return sorted(cnt, key=_u, reverse=index_order == "alphabetDesc")


def cat_to_num_unsupervised(table, list_of_cols="all", drop_cols=[], method_type="label_encoding",
                            index_order="frequencyDesc", cardinality_threshold=50, labels=None, output_mode="replace"):
    """-> (output table, {col: labels}); `labels` stands for a pre-existing StringIndexerModel."""
    cat, cols, drop = _cols(table, list_of_cols, drop_cols)
    if any(c not in cat for c in cols):
        raise TypeError("Invalid input for Column(s)")
    cols = [c for c in dict.fromkeys(cols) if c not in drop]
    cols = [c for c in cols if len(set(v for v in table.column(c).to_pylist() if v is not None)) <= cardinality_threshold]
    if not cols:
        return table, {}
    lab = labels or {c: indexer_labels(table.column(c).to_pylist(), index_order) for c in cols}
    names, arrays = list(table.column_names), [table.column(c) for c in table.column_names]
    tail_n, tail_a = [], []
    for c in cols:
        pos = {s: i for i, s in enumerate(lab[c])}
        n = len(lab[c])
        vals = table.column(c).to_pylist()
        if method_type == "label_encoding":
            arr = pa.array([None if v is None else pos.get(v, n) for v in vals], pa.int32())
            if output_mode == "replace":
                arrays[names.index(c)] = arr
            else:
                tail_n.append(c + "_index")
                tail_a.append(arr)
        else:
            idx = [n if v is None else pos.get(v, n) for v in vals]
            for j in range(n + 1):
                tail_n.append("%s_%d" % (c, j))
                tail_a.append(pa.array([int(i == j) for i in idx], pa.int32()))
    if method_type == "onehot_encoding" and output_mode == "replace":
        keep = [i for i, nme in enumerate(names) if nme not in cols]
        names, arrays = [names[i] for i in keep], [arrays[i] for i in keep]
    return pa.table(arrays + tail_a, names=names + tail_n), lab


def supervised_model(table, col, label_col, event_label):
    """The pivot of the reference: [(category | None, rate)] over the groups that have rows."""
    lab = table.column(label_col).to_pylist()
    ev = str(event_label) if pa.types.is_string(table.schema.field(label_col).type) else event_label
    g = {}
    for v, y in zip(table.column(col).to_pylist(), lab):
        a = g.setdefault(v, [0, 0])
        a[1 if (y is not None and y == ev) else 0] += 1
    tot = [sum(a[0] for a in g.values()), sum(a[1] for a in g.values())]
    if tot[0] == 0 or tot[1] == 0:
        raise ValueError("cannot resolve '%s' given input columns" % ("1" if tot[1] == 0 else "0"))
    keys = sorted(g, key=lambda k: (k is not None, _u(k) if k is not None else b""))
    return [(k, round4(g[k][1] / (g[k][0] + g[k][1]))) for k in keys]


def apply_supervised(values, model):
    if len(model) == 1:
        return [model[0][1]] * len(values)
    m = {k: v for k, v in model if k is not None}
    return [None if v is None else m.get(v) for v in values]


def cat_to_num_supervised(table, list_of_cols="all", drop_cols=[], label_col="label", event_label=1, models=None,
                          output_mode="replace"):
    """-> (output table, {col: model}); `models` stands for pre-existing saved models."""
    cat, cols, drop = _cols(table, list_of_cols, drop_cols)
    cols = [c for c in dict.fromkeys(cols) if c not in drop and c != label_col]
    if any(c not in cat for c in cols):
        raise TypeError("Invalid input for Column(s)")
    if not cols:
        return table, {}
    if label_col not in table.column_names:
        raise TypeError("Invalid input for Label Column")
    models = models or {c: supervised_model(table, c, label_col, event_label) for c in cols}
    names, arrays = list(table.column_names), [table.column(c) for c in table.column_names]
    for c in cols:
        arr = pa.array(apply_supervised(table.column(c).to_pylist(), models[c]), pa.float64())
        if output_mode == "replace":
            arrays[names.index(c)] = arr
        else:
            names.append(c + "_encoded")
            arrays.append(arr)
    return pa.table(arrays, names=names), models


def outlier_kept(values, coverage=1.0, max_category=50):
    cnt = Counter(v for v in values if v is not None)
    items = sorted(cnt.items(), key=lambda kv: (-kv[1], _u(kv[0])))
    tot = sum(cnt.values())
    kept, cumu, rank, prev = [], 0.0, 0, None
    for i, (k, n) in enumerate(items):
        if n != prev:
            rank, prev = i + 1, n
        lag = cumu
        cumu += n / tot
        if not (cumu >= coverage and lag >= coverage) and rank <= max_category - 1:
            kept.append(k)
    return kept


def outlier_categories(table, list_of_cols="all", drop_cols=[], coverage=1.0, max_category=50, params=None,
                       output_mode="replace"):
    """-> (output table, {col: kept categories}); `params` stands for a pre-existing model."""
    cat, cols, drop = _cols(table, list_of_cols, drop_cols)
    cols = [c for c in dict.fromkeys(cols) if c not in drop]
    if any(c not in cat for c in cols):
        raise TypeError("Invalid input for Column(s)")
    if not cols:
        return table, {}
    params = params if params is not None else {c: outlier_kept(table.column(c).to_pylist(), coverage, max_category)
                                                for c in cols}
    names, arrays = list(table.column_names), [table.column(c) for c in table.column_names]
    for c in cols:
        keep = set(params.get(c) or [])
        arr = pa.array([v if v is None or v in keep else "outlier_categories" for v in table.column(c).to_pylist()],
                       pa.string())
        if output_mode == "replace":
            arrays[names.index(c)] = arr
        else:
            names.append(c + "_outliered")
            arrays.append(arr)
    return pa.table(arrays, names=names), params
