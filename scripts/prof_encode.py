"""Timing of the categorical encoders on synth.device_frame(rows, cols, cat_every=1) string columns (default 40 M x 8:
two columns of each cardinality 2, 12, 100 and 10 000, Zipf-distributed codes).
  api_cold / api_warm  cat_to_num_unsupervised (label encoding of every column), cat_to_num_supervised (every other
                       column, the first card-2 column as the label) and the one-hot encoding of the card-2 and card-12
                       columns, on a fresh frame and then again (code counts from the frame's cache)
  label_pass           anv_code_map with the label-index tables (int32 out, the source's bitmap kept)
  rate_pass            anv_code_map with the supervised rate tables (double out, entry bitmaps, output bitmaps written)
  one_hot_pass         anv_one_hot of the card-2 and card-12 columns (n + 1 int32 outputs each)
  torch                the same lookups as torch composites (torch.take of the slot, the entry bitmap unpacked and
                       packed again; (idx[None] == arange(k)[:, None]).to(int32)), outputs compared bit for bit
Algorithmic bytes of a pass: one read of the codes and bitmaps, one write of the outputs (and output bitmaps); GB/s
against the 3.35 TB/s data-sheet HBM3 figure.  Prints the card and its power limit (read-only nvidia-smi query) and one
JSON line.  Usage: python scripts/prof_encode.py [rows] [cols] [reps]"""
import contextlib
import io
import json
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

sys.path.insert(0, ".")
import anovos.data_transformer.transformers as T   # noqa: E402
from anovos_b200 import engine, synth  # noqa: E402
from anovos_b200.data_transformer import transformers as TB  # noqa: E402

rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 40_000_000
ncols = int(sys.argv[2]) if len(sys.argv) > 2 else 8
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
HBM_PEAK = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def events(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _bits(words, n):
    r = torch.arange(n, device="cuda")
    return ((words[r >> 5] >> (r & 31).to(torch.int32)) & 1).bool()


def _pack(mask):
    n = mask.numel()
    m = torch.cat([mask, torch.zeros((-n) % 32, dtype=torch.bool, device="cuda")]).view(-1, 32).to(torch.int64)
    w = (m << torch.arange(32, device="cuda", dtype=torch.int64)).sum(1)
    return ((w + (1 << 31)) % (1 << 32) - (1 << 31)).to(torch.int32)


def torch_slot(fr, name):
    d, v = fr.column(name).device()
    size = len(fr.column(name).dictionary)
    s = (d.to(torch.int64) & 0xFFFFFFFF).clamp_(max=size)
    return s if v is None else torch.where(_bits(v, fr.n_rows), s, size)


def torch_map(fr, name, table, ev):
    """-> (values, output bitmap | None)."""
    s = torch_slot(fr, name)
    out = torch.take(torch.from_numpy(table).cuda(), s)
    if ev is None:
        return out, None
    keep = torch.take(torch.from_numpy(ev).cuda(), s)
    return torch.where(keep, out, torch.zeros((), dtype=out.dtype, device="cuda")), _pack(keep)


def torch_one_hot(fr, name, index, k):
    idx = torch.take(torch.from_numpy(index).cuda(), torch_slot(fr, name))
    return (idx[None] == torch.arange(k, device="cuda", dtype=torch.int32)[:, None]).to(torch.int32)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    out = {"card": card(), "rows": rows, "cols": ncols}
    quiet = contextlib.redirect_stdout(io.StringIO())
    fr = synth.device_frame(rows, ncols, seed=7, cat_every=1)
    torch.cuda.synchronize()
    names = list(fr.columns)
    by_card = {}
    for c in names:
        by_card.setdefault(len(fr.column(c).dictionary), []).append(c)
    label = by_card[min(by_card)][0]
    sup_cols = [c for c in names if c != label]
    oh_cols = [c for k in sorted(by_card)[:2] for c in by_card[k]]
    calls = {"label": lambda: T.cat_to_num_unsupervised(None, fr, list_of_cols=names, cardinality_threshold=20_000),
             "supervised": lambda: T.cat_to_num_supervised(None, fr, list_of_cols=sup_cols, label_col=label,
                                                           event_label=fr.column(label).dictionary[0]),
             "one_hot": lambda: T.cat_to_num_unsupervised(None, fr, list_of_cols=oh_cols, method_type="onehot_encoding")}
    for key, call in calls.items():
        for phase in ("cold", "warm"):
            odf = None
            t0 = time.perf_counter()
            with quiet, warnings.catch_warnings():
                warnings.simplefilter("ignore")
                odf = call()
            torch.cuda.synchronize()
            out["api_%s_%s_ms" % (key, phase)] = (time.perf_counter() - t0) * 1e3
        odf = None

    present, _ = TB._present(fr, names)
    lab_tables = [TB._label_index(fr.column(c).dictionary, TB.string_indexer_labels(present[c], "frequencyDesc"))
                  for c in names]
    allc, evc, _, _ = TB._class_counts(fr, sup_cols, label, fr.column(label).dictionary[0])
    rate = [TB._rate_table(fr.column(c).dictionary, TB._supervised_table(fr, c, allc[c], evc[c])) for c in sup_cols]
    in_bytes = {c: rows * 4 + ((rows + 7) // 8 if fr.column(c).has_validity else 0) for c in names}
    words = (rows + 31) // 32 * 4
    same = True
    for key, cols, tabs, evs, ob in (("label", names, lab_tables, [None] * len(names), 4),
                                     ("rate", sup_cols, [t for t, _ in rate], [v for _, v in rate], 8)):
        ms = events(lambda: engine.code_map(fr, cols, tabs, evs), reps)
        nbytes = sum(in_bytes[c] for c in cols) + len(cols) * rows * ob + (len(cols) * words if key == "rate" else 0)
        out[key + "_pass_ms"], out[key + "_pass_bytes"] = ms, nbytes
        out[key + "_pass_GBps"] = nbytes / ms / 1e6
        out[key + "_pass_pct_of_datasheet_3.35TBps"] = 100 * nbytes / (ms * 1e-3) / HBM_PEAK
        out[key + "_torch_ms"] = events(lambda: [torch_map(fr, c, t, e)[0].data_ptr() for c, t, e in zip(cols, tabs, evs)],
                                        reps)
        data, valid, _ = engine.code_map(fr, cols, tabs, evs)
        for i, (c, t, e) in enumerate(zip(cols, tabs, evs)):
            y, vw = torch_map(fr, c, t, e)
            same = same and torch.equal(data[i].view(torch.uint8), y.view(torch.uint8))
            if vw is not None:
                same = same and torch.equal(valid[i], vw)
        del data, valid
    idx = [lab_tables[names.index(c)] for c in oh_cols]
    ks = [int(ix.max()) + 1 for ix in idx]
    ms = events(lambda: engine.one_hot(fr, oh_cols, idx, ks), reps)
    nbytes = sum(in_bytes[c] for c in oh_cols) + sum(ks) * rows * 4
    out["one_hot_k"], out["one_hot_pass_ms"], out["one_hot_pass_bytes"] = ks, ms, nbytes
    out["one_hot_pass_GBps"] = nbytes / ms / 1e6
    out["one_hot_pass_pct_of_datasheet_3.35TBps"] = 100 * nbytes / (ms * 1e-3) / HBM_PEAK
    outs = engine.one_hot(fr, oh_cols, idx, ks)
    for o, c, ix, k in zip(outs, oh_cols, idx, ks):
        same = same and torch.equal(o, torch_one_hot(fr, c, ix, k))
    del outs
    out["one_hot_torch_ms"] = events(lambda: [torch_one_hot(fr, c, ix, k).data_ptr() for c, ix, k in zip(oh_cols, idx, ks)],
                                     reps)
    out["bit_identical"] = bool(same)
    print(json.dumps(out))


if __name__ == "__main__":
    np.seterr(all="ignore")
    main()
