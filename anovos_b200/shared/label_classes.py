"""Label classes of a frame as validity bitmaps, shared by IV / IG (data_analyzer.association_evaluator) and the
supervised categorical encoder (data_transformer.transformers.cat_to_num_supervised): a per-category count of the rows of
one class is the code histogram of a view whose validity is AND-ed with the class bitmap."""
from __future__ import annotations

from collections import OrderedDict

from ..frame import Column, ColumnFrame


def _pack_bits(mask):
    """bool CUDA tensor [n] -> int32 Arrow bitmap words (LSB-first)."""
    import torch
    n = mask.numel()
    pad = (-n) % 32
    if pad:
        mask = torch.cat([mask, torch.zeros(pad, dtype=torch.bool, device=mask.device)])
    w = (mask.view(-1, 32).to(torch.int64) << torch.arange(32, device=mask.device, dtype=torch.int64)).sum(dim=1)
    return ((w + (1 << 31)) % (1 << 32) - (1 << 31)).to(torch.int32)


def _unpack_bits(words, n):
    import torch
    rows = torch.arange(n, device=words.device)
    return ((words[rows >> 5] >> (rows & 31).to(torch.int32)) & 1).bool()


def label_bitmaps(fr: ColumnFrame, label_col, event_label):
    """-> (event words, non-event words, n_event): rows with label == event_label / label != event_label
    (a null label is in neither class)."""
    import torch
    col = fr.column(label_col)
    d, v = col.device()
    if col.kind == "cat":
        try:
            code = col.dictionary.index(str(event_label))
        except ValueError:
            code = -1
        is_ev = d == code
    else:
        is_ev = d.to(torch.float64) == float(event_label)
    valid = _unpack_bits(v, fr.n_rows) if v is not None else torch.ones(fr.n_rows, dtype=torch.bool, device=d.device)
    ev, nev = is_ev & valid, (~is_ev) & valid
    return _pack_bits(ev), _pack_bits(nev), int(ev.sum().item())


def masked(fr: ColumnFrame, names, words) -> ColumnFrame:
    """Same columns with validity := validity AND words (rows outside the class become "null")."""
    cols = OrderedDict()
    for n in names:
        c = fr.column(n)
        d, v = c.device()
        nv = words if v is None else (v & words)
        cols[n] = Column(n, c.sdtype, fr.n_rows, dev=d, dev_valid=nv, anv_dtype=c.anv_dtype, dictionary=c.dictionary)
    return ColumnFrame(cols, fr.n_rows)
