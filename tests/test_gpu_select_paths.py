"""GPU tests of the radix select's refinement passes (csrc/select.cu) on the slot-table paths quantile-chosen ranks reach
only by chance, against exact order statistics.

After pass 0 a pass counts a value only if its decided prefix is one of <= 16 target slots, found through a 4096-cell byte
table indexed by prefix_hash.  The first slot wins a cell; a second target in the same cell, and a value whose prefix is no
target but hashes to a used cell (a foreign prefix), take the linear search.  The columns here are built in key space so
that those cases happen at a chosen pass of every key type: colliding targets whose later slot holds the most values,
foreign prefixes below and above the targets (one outnumbering its target 1 000 to 1), 16 slots (the 64 KB histogram),
16 ranks in one slot, skipped / repeated / end ranks, 40 ranks over both key widths, a colliding prefix held only by the
scalar tail, nulls across bitmap words, one value filling a tile, and the per-partition protocol over uneven chunks.

The module restates the kernel's order-preserving key, its pass geometry and prefix_hash, and replays the selection on
the host (`replay`).  Every test asserts through the replay the geometry it relies on (the pass and the slots that
collide, the foreign counts), and that the two ways to get the slow path wrong - dropping the values that miss their
cell's first slot, or counting everything in a used cell into it - would change the values it checks.  The expected
values are the exact reference: the valid values sorted (NaN last, -0.0 == 0.0, integers sorted exactly), srt[k - 1]."""
import numpy as np
import pytest

from test_gpu_kernel_edges import _same_float

pytestmark = pytest.mark.gpu

# ---- restatement of select.cu ------------------------------------------------------------------------------------

SEL_BITS0, SEL_BITS, SEL_MAX_RANKS = 12, 10, 16      # digit widths of pass 0 / later passes, ranks per call
HASH_LO, HASH_HI = 0x9E3779B1, 0x85EBCA77            # prefix_hash multipliers of the low / high 32 prefix bits
CELLS = 1 << SEL_BITS0                               # cells of the slot table
TILE_MIN, TILE_MAX = 32768, 1 << 20                  # sel_tile_rows bounds
KEY_BITS = {"f32": 32, "i32": 32, "f64": 64, "i64": 64}
VEC = {"f32": 4, "i32": 4, "f64": 2, "i64": 2}          # values per 16-byte load; the rest of a tile is the scalar tail
NP = {"f32": np.float32, "i32": np.int32, "f64": np.float64, "i64": np.int64}
U64 = np.uint64
ALL_PASSES = [(dt, p) for dt in ("f32", "i32") for p in (1, 2)] + [(dt, p) for dt in ("f64", "i64") for p in range(1, 7)]


def pass_geometry(key_bits):
    """[(bits, shift, decided)] of every pass: 12 bits, then 10 at a time (3 passes for 32-bit keys, 7 for 64-bit keys,
    the last of those taking 2 bits).  digit = (key >> shift) & (2^bits - 1); the prefix a pass matches is key >> (64 - decided)."""
    out, decided = [], 0
    while decided < key_bits:
        b = SEL_BITS0 if not out else min(SEL_BITS, key_bits - decided)
        out.append((b, 64 - decided - b, decided))
        decided += b
    return out


def sort_key(x, dt):
    """The kernel's order-preserving key as uint64 (32-bit keys in the high half): -0.0 is 0.0, every NaN sorts last."""
    x = np.atleast_1d(np.asarray(x, NP[dt]))
    w = KEY_BITS[dt]
    if dt in ("f32", "f64"):
        full = U64((1 << w) - 1)
        sign = U64(1 << (w - 1))
        u = x.view(np.uint32 if w == 32 else U64).astype(U64)
        u = np.where(u == sign, U64(0), u)                                 # x + 0.0
        k = np.where(u & sign, ~u & full, u | sign)
        k = np.where(np.isnan(x), full, k)
    elif dt == "i32":
        k = (x.view(np.uint32) ^ np.uint32(0x80000000)).astype(U64)
    else:
        k = x.view(U64) ^ U64(1 << 63)
    return np.asarray(k, U64) << U64(64 - w)


def key_value(k, dt):
    """Inverse of sort_key (key_to_double before the conversion to double): the value of each key."""
    w = KEY_BITS[dt]
    k = np.asarray(k, U64) >> U64(64 - w)
    if dt in ("f32", "f64"):
        sign = U64(1 << (w - 1))
        u = np.where(k & sign, k & ~sign, ~k & U64((1 << w) - 1))
        return u.astype(np.uint32).view(np.float32) if w == 32 else u.view(np.float64)
    if dt == "i32":
        return (k.astype(np.uint32) ^ np.uint32(0x80000000)).view(np.int32)
    return (k ^ U64(1 << 63)).view(np.int64)


def valid_keys(k, dt):
    """Keys that are the key of their own value (not a NaN other than the last key, not -0.0)."""
    return sort_key(key_value(k, dt), dt) == np.asarray(k, U64)


def prefix_hash(pf):
    """12-bit cell of each right-aligned prefix."""
    pf = np.atleast_1d(np.asarray(pf, U64))
    m = U64(0xFFFFFFFF)
    x = ((pf & m) * U64(HASH_LO) + (pf >> U64(32)) * U64(HASH_HI)) & m
    return (x >> U64(32 - SEL_BITS0)).astype(np.int64)


def replay(keys, ranks, key_bits, mode="exact"):
    """The selection of select_pass_kernel / select_scan_kernel on the host.  keys: sort_key of the valid values; ranks:
    1-based (0 = skip).  mode "exact" is the kernel; "drop" counts a value only when its prefix is its cell's first slot
    (no linear search), "cell" counts every value of a used cell into the cell's first slot (no prefix compare).
    -> (64-bit key of each selected value, None where skipped;  one record per pass: its geometry, the slot prefixes,
    each rank's slot, each slot's cell and the slot that won it, the slots that lost their cell, the values counted per
    slot and the foreign values in each slot's cell)."""
    keys = np.asarray(keys, U64)
    rank = [int(r) for r in ranks]
    prefix = [0] * len(rank)
    passes = []
    for p, (bits, shift, decided) in enumerate(pass_geometry(key_bits)):
        nb = 1 << bits
        digit = ((keys >> U64(shift)) & U64(nb - 1)).astype(np.int64)
        slot_prefix, rank_slot = [], [-1] * len(rank)
        for i, r in enumerate(rank):
            if r > 0:
                if prefix[i] not in slot_prefix:
                    slot_prefix.append(prefix[i])
                rank_slot[i] = slot_prefix.index(prefix[i])
        rec = dict(index=p, bits=bits, shift=shift, decided=decided, slot_prefix=slot_prefix, rank_slot=rank_slot)
        ns = len(slot_prefix)
        if p == 0:
            slot = np.zeros(keys.size, np.int64) if ns else np.full(keys.size, -1, np.int64)
        else:
            pf = keys >> U64(64 - decided)
            cells = prefix_hash(np.array(slot_prefix, U64)) if ns else np.zeros(0, np.int64)
            tbl = np.full(CELLS, -1, np.int64)
            for q in range(ns):
                if tbl[cells[q]] < 0:
                    tbl[cells[q]] = q
            cand = tbl[prefix_hash(pf)] if keys.size else np.zeros(0, np.int64)
            own = np.full(keys.size, -1, np.int64)
            for q, s in enumerate(slot_prefix):
                own[pf == U64(s)] = q
            slot = {"exact": own, "drop": np.where(own == cand, own, -1), "cell": cand}[mode]
            rec.update(cells=cells.tolist(), winner=[int(tbl[c]) for c in cells],
                       losers=[q for q in range(ns) if tbl[cells[q]] != q],
                       counted=np.bincount(own[own >= 0], minlength=ns)[:ns].tolist(),
                       foreign=[int(((cand == tbl[cells[q]]) & (own < 0)).sum()) for q in range(ns)])
        for i, r in enumerate(rank):
            if r <= 0:
                continue
            cum = np.cumsum(np.bincount(digit[slot == rank_slot[i]], minlength=nb))
            d = min(int(np.searchsorted(cum, r, "left")), nb - 1)    # first bin with cum >= rank; the last one if none
            rank[i] = r - (int(cum[d - 1]) if d else 0)
            prefix[i] = (prefix[i] << bits) | d
        passes.append(rec)
    return [U64(prefix[i]) << U64(64 - key_bits) if r > 0 else None for i, r in enumerate(ranks)], passes


def replay_values(vals, valid, ranks, dt, mode="exact"):
    """float64 values the kernel reports for `ranks` (NaN where skipped), and the pass records."""
    sel, passes = replay(sort_key(vals[valid], dt), ranks, KEY_BITS[dt], mode)
    return np.array([np.nan if k is None else float(key_value(k, dt)) for k in sel]), passes


def reference(vals, valid, ranks):
    x = vals[valid]
    srt = np.sort(x.astype(np.float64) if x.dtype.kind == "f" else x)     # NaN last; integers sorted exactly
    return np.array([float(srt[k - 1]) if k else np.nan for k in ranks])


def tile_rows(n_rows, n_cols, sms):
    """sel_tile_rows: rows per CTA of a column."""
    per_col = -(-sms * 4 // max(n_cols, 1))
    tr = n_rows // per_col
    t = TILE_MIN
    while t < tr and t < TILE_MAX:
        t <<= 1
    return t


# ---- columns built in key space -----------------------------------------------------------------------------------

def _region(dt, decided):
    """Key ranges [lo, hi) the candidate prefixes of a pass come from: the whole key space for 32-bit integers; floats of
    magnitude 2^-8 .. 2^24 of either sign; int64 within 2^(84 - decided) of 0, so that the prefixes are spread well
    beyond 4 096 consecutive values (the hash spreads a run of consecutive prefixes evenly) while a wrong digit of the
    pass still changes the value as a double."""
    if dt == "i32":
        return [(0, 1 << 64)]
    if dt == "i64":
        hw = 1 << min(63, 84 - decided)
        return [((1 << 63) - hw, (1 << 63) + hw)]
    lo, hi = (int(sort_key(v, dt)[0]) for v in (2.0 ** -8, 2.0 ** 24))
    nlo, nhi = (int(sort_key(v, dt)[0]) for v in (-2.0 ** 24, -2.0 ** -8))
    return [(nlo, nhi), (lo, hi)]


def _random_keys(dt, n, rng, region):
    out = []
    for lo, hi in region:
        span = hi - lo
        r = rng.integers(0, 1 << 62, size=2 * n, dtype=U64).astype(object)   # exact big-int scaling into [lo, hi)
        out.append(np.array([lo + int(v) * span // (1 << 62) for v in r], dtype=U64))
    k = np.concatenate(out) & ~U64((1 << (64 - KEY_BITS[dt])) - 1)
    k = k[valid_keys(k, dt)]
    return rng.permutation(k)[:n]


def candidates(dt, decided, rng):
    """Sorted prefixes (right-aligned, `decided` bits) of valid keys: every 12-bit prefix whose keys are all values at
    pass 1, prefixes of random keys of the type's region later."""
    w = KEY_BITS[dt]
    if decided == SEL_BITS0:
        pf = np.arange(CELLS, dtype=U64)
        low = U64(64 - decided)
        last = (pf << low) | (((U64(1) << low) - U64(1)) & ~U64((1 << (64 - w)) - 1))
        return pf[valid_keys(pf << low, dt) & valid_keys(last, dt)]
    return np.unique(_random_keys(dt, 40_000, rng, _region(dt, decided)) >> U64(64 - decided))


def cells_of(dt, decided, rng, need):
    """Cells of the slot table holding at least `need` candidate prefixes -> (candidates, their cells, those cells).
    At pass 1 no cell holds more than two of the 4 096 prefixes."""
    pf = candidates(dt, decided, rng)
    h = prefix_hash(pf)
    full = np.flatnonzero(np.bincount(h, minlength=CELLS) >= need)
    assert full.size, (dt, decided, need)
    return pf, h, full


def colliding_cell(dt, decided, rng, need=4):
    """`need` or more sorted prefixes of one cell of the slot table (a random cell among those holding as many)."""
    pf, h, full = cells_of(dt, decided, rng, need)
    cell = rng.choice(full)
    return [int(v) for v in np.sort(pf[h == cell])]


def block(dt, prefix, decided, n, rng):
    """n valid keys under `prefix` (right-aligned, `decided` bits), low bits uniform."""
    low = KEY_BITS[dt] - decided
    base = prefix << (64 - decided)
    r = rng.integers(0, 1 << low, size=2 * n + 8, dtype=U64) if low < 64 else rng.integers(0, 1 << 63, 2 * n + 8, U64)
    k = U64(base) | (r << U64(64 - KEY_BITS[dt]))
    k = k[valid_keys(k, dt)][:n]
    assert k.size == n
    return k


def null_mask(n, rng, rate=0.04):
    """Random nulls plus runs of 8 nulls across every fourth bitmap word boundary (rows 28 .. 35 of each 128)."""
    r = np.arange(n)
    return (rng.random(n) < rate) | ((r % 128 >= 28) & (r % 128 < 36))


def in_prefix(keys, prefix, decided):
    return (np.asarray(keys, U64) >> U64(64 - decided)) == U64(prefix)


class Case:
    """One column: values, validity, the ranks asked of it and what it was built to show."""

    def __init__(self, name, dt, keys, valid, ranks, **info):
        self.name, self.dt, self.valid, self.ranks, self.info = name, dt, np.asarray(valid, bool), list(ranks), info
        self.keys = np.asarray(keys, U64)
        self.vals = key_value(self.keys, dt)

    def expected(self):
        return reference(self.vals, self.valid, self.ranks)

    def replay(self, mode="exact"):
        return replay_values(self.vals, self.valid, self.ranks, self.dt, mode)


def _shuffle(rng, keys, valid):
    o = rng.permutation(keys.size)
    return keys[o], valid[o]


def digit_of(keys, key_bits, p):
    bits, shift, _ = pass_geometry(key_bits)[p]
    return (np.atleast_1d(np.asarray(keys, U64)) >> U64(shift)) & U64((1 << bits) - 1)


def _ranks_in(sorted_keys, prefix, decided, fracs, key_bits=None, p=None):
    """1-based ranks at fractions of the run of sorted valid keys under `prefix`.  Given a pass, each rank moves down to a
    value whose digit of that pass is not the largest: an empty slot histogram resolves a rank to the largest digit, so
    at the last pass a value with that digit would come out right even from a slot that counted nothing."""
    lo = int(np.searchsorted(sorted_keys >> U64(64 - decided), U64(prefix), "left"))
    hi = int(np.searchsorted(sorted_keys >> U64(64 - decided), U64(prefix), "right"))
    assert hi > lo
    out = []
    for f in fracs:
        r = lo + 1 + min(int(f * (hi - lo)), hi - lo - 1)
        if p is not None:
            top = U64((1 << pass_geometry(key_bits)[p][0]) - 1)
            while r > lo + 1 and digit_of(sorted_keys[r - 1], key_bits, p)[0] == top:
                r -= 1
        out.append(r)
    return out


def collision_case(dt, p, seed, n_a=3000, n_b=9000, n_f=4000, n_bg=20000, null_rows=4000):
    """Targets in two prefixes A < B that share a cell at pass p (A's ranks first, so A's slot wins the cell and B's,
    the one holding the most values, takes the linear search), foreign prefixes below A and above B in the cell of a
    target, a background, and nulls hiding B-prefix values.  From pass 2 on the foreign prefixes share A's cell; at
    pass 1, whose cells hold two prefixes at most, each is the partner of a target C of its own cell."""
    rng = np.random.default_rng(seed)
    decided = pass_geometry(KEY_BITS[dt])[p][2]
    if p > 1:
        cell = colliding_cell(dt, decided, rng)
        a, b = cell[1], cell[2]
        foreign = [(a, cell[0]), (a, cell[-1])]
    else:
        pf, h, full = cells_of(dt, decided, rng, 2)
        pairs = [sorted(int(v) for v in pf[h == c]) for c in rng.permutation(full)]
        a, b = next(q for q in pairs if q[0] > pf[pf.size // 8] and q[1] < pf[-pf.size // 8])
        lo = next(q for q in pairs if q[0] < a and q != [a, b])
        hi = next(q for q in pairs if q[1] > b and q not in ([a, b], lo))
        foreign = [(lo[1], lo[0]), (hi[0], hi[1])]
    used = {a, b} | {x for pair in foreign for x in pair}
    bg = _random_keys(dt, n_bg, rng, _region(dt, decided))
    bg = bg[~np.isin(bg >> U64(64 - decided), np.array(sorted(used), U64))]
    targets = [block(dt, a, decided, n_a, rng), block(dt, b, decided, n_b, rng)]
    targets += [block(dt, t, decided, n_f // 8, rng) for t, _ in foreign if t != a]
    foreign_keys = [block(dt, f, decided, n_f // 2, rng) for _, f in foreign]
    valid_keys_ = np.concatenate(targets + foreign_keys + [bg])
    keys = np.concatenate([valid_keys_, block(dt, b, decided, null_rows, rng)])
    valid = np.concatenate([np.ones(valid_keys_.size, bool), np.zeros(null_rows, bool)])
    keys, valid = _shuffle(rng, keys, valid)
    srt = np.sort(keys[valid])
    ranks = _ranks_in(srt, a, decided, (0.35, 0.7), KEY_BITS[dt], p) + _ranks_in(srt, b, decided, (0.2, 0.5, 0.9), KEY_BITS[dt], p)
    ranks += [_ranks_in(srt, t, decided, (0.6,), KEY_BITS[dt], p)[0] for t, _ in foreign if t != a]
    return Case("%s_pass%d" % (dt, p), dt, keys, valid, ranks, p=p, decided=decided, a=a, b=b, foreign=foreign,
                n_foreign=n_f // 2)


def assert_collision(case, passes):
    """Pass p has A and B as its slots, in one cell, and B (holding the most values) takes the linear search."""
    rec = passes[case.info["p"]]
    a, b = case.info["a"], case.info["b"]
    assert rec["decided"] == case.info["decided"]
    assert a in rec["slot_prefix"] and b in rec["slot_prefix"], rec["slot_prefix"]
    qa, qb = rec["slot_prefix"].index(a), rec["slot_prefix"].index(b)
    assert qa < qb and rec["cells"][qa] == rec["cells"][qb], rec
    assert qb in rec["losers"] and rec["winner"][qb] == qa, rec
    return rec, qa, qb


def assert_would_change(case, exp, modes=("drop", "cell"), where=None):
    """The replay of a slot table without the linear search ("drop") or without the prefix compare ("cell") gives other
    values at the ranks `where` (every rank by default): a kernel taking either shortcut fails the test."""
    where = np.arange(len(case.ranks)) if where is None else np.asarray(where)
    for mode in modes:
        got, _ = case.replay(mode)
        same = [i for i in where if _same_float(got[i], exp[i])]
        assert not same, (case.name, mode, same)


# ---- GPU helpers ------------------------------------------------------------------------------------------------------

def frame_of(cases, n=None):
    """ColumnFrame of the cases' columns, each padded with null rows to n rows.  Values under nulls stay as built."""
    from anovos_b200.frame import ColumnFrame, _pack_validity
    n = max(c.keys.size for c in cases) if n is None else n
    data = {}
    for c in cases:
        pad = n - c.keys.size
        vals = np.concatenate([c.vals, np.resize(c.vals, pad)]) if pad else c.vals
        valid = np.concatenate([c.valid, np.zeros(pad, bool)])
        data[c.name] = (np.ascontiguousarray(vals), None if valid.all() else _pack_validity(valid))
    return ColumnFrame.from_tensors(data, n_rows=n)


def rank_matrix(cases, width=None):
    width = max(len(c.ranks) for c in cases) if width is None else width
    rk = np.zeros((len(cases), width), np.int64)
    for i, c in enumerate(cases):
        rk[i, :len(c.ranks)] = c.ranks
    return rk


def select(fr, cases, rk=None):
    from anovos_b200 import engine
    rk = rank_matrix(cases) if rk is None else rk
    return engine.select_ranks(fr, [c.name for c in cases], rk)


def check(cases, got):
    for i, c in enumerate(cases):
        exp = c.expected()
        assert _same_float(got[i, :len(c.ranks)], exp), (c.name, got[i, :len(c.ranks)], exp)
        assert np.isnan(got[i, len(c.ranks):]).all()


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- 2 / 3: colliding targets and foreign prefixes at every refinement pass ------------------------------------------

@pytest.fixture(scope="module")
def collision_cases():
    return [collision_case(dt, p, seed=100 + 10 * i) for i, (dt, p) in enumerate(ALL_PASSES)]


@pytest.mark.parametrize("dt,p", ALL_PASSES, ids=["%s-pass%d" % a for a in ALL_PASSES])
def test_colliding_targets(dt, p, collision_cases):
    """Ranks in two prefixes of one cell at pass p: the later slot, with three times the values, is found only by the
    linear search.  Dropping its values would move every one of its ranks."""
    case = collision_cases[ALL_PASSES.index((dt, p))]
    exp = case.expected()
    got_r, passes = case.replay()
    assert _same_float(got_r, exp)
    rec, qa, qb = assert_collision(case, passes)
    assert rec["counted"][qb] > rec["counted"][qa]
    assert_would_change(case, exp, ("drop",), where=[i for i, s in enumerate(rec["rank_slot"]) if s == qb])
    fr = frame_of([case])
    assert tile_rows(fr.n_rows, 1, _sms()) < fr.n_rows                   # the column spans several tiles
    check([case], select(fr, [case]))


def test_colliding_targets_in_one_call(collision_cases):
    """All the collision columns in one call: four 32-bit and twelve 64-bit columns, two tiles each."""
    fr = frame_of(collision_cases)
    assert tile_rows(fr.n_rows, 4, _sms()) < fr.n_rows and tile_rows(fr.n_rows, 12, _sms()) < fr.n_rows
    check(collision_cases, select(fr, collision_cases))


@pytest.mark.parametrize("dt,p", ALL_PASSES, ids=["%s-pass%d" % a for a in ALL_PASSES])
def test_foreign_prefixes_in_used_cells(dt, p, collision_cases):
    """The same columns hold foreign prefixes below A and above B in a target's cell (and B's values are foreign to A's
    slot): counting what lands in a used cell into its first slot would change every selected value."""
    case = collision_cases[ALL_PASSES.index((dt, p))]
    exp = case.expected()
    _, passes = case.replay()
    rec, qa, qb = assert_collision(case, passes)
    (_, f_lo), (_, f_hi) = case.info["foreign"]
    assert f_lo < case.info["a"] < case.info["b"] < f_hi
    for t, f in case.info["foreign"]:
        q = rec["slot_prefix"].index(t)
        assert f not in rec["slot_prefix"] and prefix_hash(f)[0] == rec["cells"][q]
        assert rec["foreign"][q] >= case.info["n_foreign"], rec
    assert_would_change(case, exp, ("cell",))
    check([case], select(frame_of([case]), [case]))


def foreign_heavy_case(dt, p, seed):
    """Target A (12 values) and foreign prefixes of its cell holding 12 000 values: one on each side of A, or at pass 1
    (two prefixes to a cell) A's partner."""
    rng = np.random.default_rng(seed)
    decided = pass_geometry(KEY_BITS[dt])[p][2]
    cell = colliding_cell(dt, decided, rng, need=2 if p == 1 else 3)
    a = cell[1]
    fs = [f for f in cell if f != a][:2]
    keys = np.concatenate([block(dt, a, decided, 12, rng)] + [block(dt, f, decided, 12000 // len(fs), rng) for f in fs]
                          + [_random_keys(dt, 3000, rng, _region(dt, decided))])
    keys = keys[~(in_prefix(keys, a, decided) & (np.arange(keys.size) >= 12))]     # A holds exactly its 12 values
    valid = np.ones(keys.size, bool)
    keys, valid = _shuffle(rng, keys, valid)
    ranks = _ranks_in(np.sort(keys), a, decided, (0.25, 0.5, 0.99))
    return Case("heavy_%s_pass%d" % (dt, p), dt, keys, valid, ranks, p=p, decided=decided, a=a)


HEAVY = [(dt, p) for dt in ("f32", "i32", "f64", "i64") for p in (1, len(pass_geometry(KEY_BITS[dt])) - 1)]


@pytest.mark.parametrize("dt,p", HEAVY, ids=["%s-pass%d" % a for a in HEAVY])
def test_foreign_prefix_outnumbers_target_1000_to_1(dt, p):
    case = foreign_heavy_case(dt, p, seed=300 + HEAVY.index((dt, p)))
    exp = case.expected()
    got_r, passes = case.replay()
    assert _same_float(got_r, exp)
    rec = passes[p]
    assert rec["slot_prefix"] == [case.info["a"]] and rec["counted"] == [12]
    assert rec["foreign"][0] >= 1000 * rec["counted"][0], rec
    assert_would_change(case, exp, ("cell",))
    check([case], select(frame_of([case]), [case]))


# ---- 4: slot-table extremes ---------------------------------------------------------------------------------------------

def sixteen_slots_case(dt, seed):
    """16 ranks in 16 distinct pass-1 prefixes, hence 16 slots at every refinement pass (16 x 1024 x 4 B of shared
    histogram); two of the prefixes share a cell at pass 1."""
    rng = np.random.default_rng(seed)
    pair = colliding_cell(dt, SEL_BITS0, rng, need=2)[:2]
    rest = rng.choice(np.setdiff1d(candidates(dt, SEL_BITS0, rng), np.array(pair, U64)), 14, replace=False)
    pfs = [int(v) for v in pair] + [int(v) for v in rest]
    keys = np.concatenate([block(dt, q, SEL_BITS0, 300 + 40 * i, rng) for i, q in enumerate(pfs)])
    valid = ~null_mask(keys.size, rng)
    keys, valid = _shuffle(rng, keys, valid)
    srt = np.sort(keys[valid])
    ranks = [_ranks_in(srt, q, SEL_BITS0, (0.6,))[0] for q in pfs]
    return Case("slots16_" + dt, dt, keys, valid, ranks)


def one_slot_case(dt, seed):
    """16 adjacent ranks that share one prefix down to the last pass: a run of 10 equal values among single keys of the
    same last-pass prefix (consecutive keys for 32-bit types; the four keys of a 2-bit last digit for 64-bit types)."""
    rng = np.random.default_rng(seed)
    bits, _, last = pass_geometry(KEY_BITS[dt])[-1]
    pf = candidates(dt, last, rng)
    step = U64(1) << U64(64 - KEY_BITS[dt])
    base = U64(int(pf[pf.size // 2])) << U64(64 - last)                # first key of a last-pass prefix
    if bits == SEL_BITS:
        near, counts, first = base + step * (U64(8) + np.arange(11, dtype=U64)), [1] * 5 + [10] + [1] * 5, 2
    else:
        near, counts, first = base + step * np.arange(4, dtype=U64), [2, 10, 1, 3], 0
    assert valid_keys(near, dt).all()
    bg = _random_keys(dt, 5000, rng, _region(dt, last))
    keys = np.concatenate([np.repeat(near, counts), bg[~in_prefix(bg, int(pf[pf.size // 2]), last)]])
    valid = np.ones(keys.size, bool)
    keys, valid = _shuffle(rng, keys, valid)
    lo = int(np.searchsorted(np.sort(keys), near[first]))
    return Case("slot1_" + dt, dt, keys, valid, range(lo + 1, lo + 17), last=last)


def edge_ranks_case(dt, seed):
    """Skipped ranks (0) among repeated ranks, rank 1 and rank n_valid, on a collision column."""
    base = collision_case(dt, 1, seed, n_a=500, n_b=1500, n_f=600, n_bg=3000, null_rows=500)
    n_valid = int(base.valid.sum())
    ra, rb = base.ranks[0], base.ranks[3]
    ranks = [0, 1, ra, rb, 0, n_valid, rb, ra, 0, rb, 1, n_valid, 0, rb, 0, 0]
    return Case("edge_" + dt, dt, base.keys, base.valid, ranks, **base.info)


@pytest.mark.parametrize("dt", ["f32", "i32", "f64", "i64"])
def test_sixteen_distinct_slots_through_every_pass(dt):
    case = sixteen_slots_case(dt, seed=400 + len(dt) + ord(dt[0]))
    exp = case.expected()
    got_r, passes = case.replay()
    assert _same_float(got_r, exp)
    assert all(len(rec["slot_prefix"]) == SEL_MAX_RANKS for rec in passes[1:])
    assert SEL_MAX_RANKS * (1 << SEL_BITS) * 4 > 40 * 1024                 # the shared histogram takes the opt-in
    assert passes[1]["losers"], passes[1]["cells"]
    check([case], select(frame_of([case]), [case]))


@pytest.mark.parametrize("dt", ["f32", "i32", "f64", "i64"])
def test_sixteen_ranks_in_one_slot_to_the_last_pass(dt):
    case = one_slot_case(dt, seed=500 + ord(dt[0]) + int(dt[1:]))
    exp = case.expected()
    got_r, passes = case.replay()
    assert _same_float(got_r, exp)
    assert all(len(rec["slot_prefix"]) == 1 and set(rec["rank_slot"]) == {0} for rec in passes)
    assert np.unique(exp).size == min(7, 1 << passes[-1]["bits"]) and (np.diff(exp) == 0).sum() >= 9
    check([case], select(frame_of([case]), [case]))


def test_skipped_repeated_and_end_ranks():
    """One call over both key widths: 0 ranks mixed in, repeated ranks sharing a slot, rank 1 and rank n_valid, and a
    column whose every rank is 0."""
    cases = [edge_ranks_case(dt, 600 + i) for i, dt in enumerate(("f32", "i32", "f64", "i64"))]
    skip = collision_case("f64", 2, 650, n_a=100, n_b=200, n_f=100, n_bg=500, null_rows=50)
    cases.append(Case("none", "f64", skip.keys, skip.valid, [0] * 16))
    for c in cases[:4]:
        exp = c.expected()
        got_r, passes = c.replay()
        assert _same_float(got_r, exp)
        rk = np.array(c.ranks)
        assert np.isnan(exp[rk == 0]).all() and (rk == 0).sum() == 6
        assert all(np.unique(exp[rk == r]).size == 1 for r in rk) and {1, int(c.valid.sum())} <= set(c.ranks)
        assert_collision(c, passes)
    got = select(frame_of(cases), cases)
    check(cases, got)
    assert np.isnan(got[-1]).all()


def forty_ranks_cases():
    """f32, f64, i32 and i64 collision columns with 40 ranks each, the collision ranks in every group of 16."""
    out = []
    for i, (dt, p) in enumerate((("f32", 2), ("f64", 3), ("i32", 1), ("i64", 5), ("f64", 6), ("f32", 1))):
        c = collision_case(dt, p, 700 + i, n_a=800, n_b=2400, n_f=800, n_bg=6000, null_rows=300)
        rng = np.random.default_rng(750 + i)
        n_valid = int(c.valid.sum())
        ranks = list(rng.integers(1, n_valid + 1, 40))
        for g in range(3):                                   # the five collision ranks lead every group of 16
            ranks[16 * g:16 * g + 5] = c.ranks
        out.append(Case("r40_%s_pass%d" % (dt, p), dt, c.keys, c.valid, ranks, **c.info))
    return out


def test_forty_ranks_over_both_key_widths():
    cases = forty_ranks_cases()
    rk = rank_matrix(cases)
    assert rk.shape[1] > 2 * SEL_MAX_RANKS and {KEY_BITS[c.dt] for c in cases} == {32, 64}
    for c in cases:
        for g in range(3):                                   # every group of 16 ranks sees the collision at its pass
            part = Case(c.name, c.dt, c.keys, c.valid, c.ranks[16 * g:16 * g + 16], **c.info)
            assert_collision(part, part.replay()[1])
    check(cases, select(frame_of(cases), cases, rk))


# ---- 5: tile geometry ----------------------------------------------------------------------------------------------------

TAIL = [(dt, p) for dt in ("f32", "i32", "f64", "i64") for p in (1, len(pass_geometry(KEY_BITS[dt])) - 1)]


def tail_case(dt, p, seed, tiles=3):
    """A column of several tiles and n % VEC rows past its last full vector; B, the prefix that collides with target A at
    pass p, is held only by those scalar-tail rows (one of them null when the tail has more than one row)."""
    rng = np.random.default_rng(seed)
    vec = VEC[dt]
    n = TILE_MIN * tiles + 1000 * vec + vec - 1
    decided = pass_geometry(KEY_BITS[dt])[p][2]
    a, b = colliding_cell(dt, decided, rng, need=2)[:2]
    tail = block(dt, b, decided, 8 * vec, rng)
    tail = tail[digit_of(tail, KEY_BITS[dt], p) < U64((1 << pass_geometry(KEY_BITS[dt])[p][0]) - 1)][:vec - 1]
    body = np.concatenate([block(dt, a, decided, 2000, rng), _random_keys(dt, n - 2000 - (vec - 1), rng, _region(dt, decided))])
    body = body[~in_prefix(body, b, decided)]
    body = np.concatenate([body, block(dt, a, decided, n - (vec - 1) - body.size, rng)])
    body_valid = ~null_mask(body.size, rng)
    body, body_valid = _shuffle(rng, body, body_valid)
    keys = np.concatenate([body, tail])
    valid = np.concatenate([body_valid, np.arange(vec - 1) != 1])
    srt = np.sort(keys[valid])
    ranks = _ranks_in(srt, a, decided, (0.5,)) + _ranks_in(srt, b, decided, (0.0, 0.99))
    return Case("tail_%s_pass%d" % (dt, p), dt, keys, valid, ranks, p=p, decided=decided, a=a, b=b)


@pytest.mark.parametrize("dt,p", TAIL, ids=["%s-pass%d" % a for a in TAIL])
def test_colliding_prefix_only_in_the_scalar_tail(dt, p):
    case = tail_case(dt, p, seed=800 + TAIL.index((dt, p)))
    n, vec = case.keys.size, VEC[dt]
    tr = tile_rows(n, 1, _sms())
    assert n // tr >= 3 and n % tr % vec == vec - 1                         # several tiles; the last has a scalar tail
    holders = np.flatnonzero(in_prefix(case.keys, case.info["b"], case.info["decided"]))
    assert holders.min() >= n - n % vec
    exp = case.expected()
    got_r, passes = case.replay()
    assert _same_float(got_r, exp)
    rec, qa, qb = assert_collision(case, passes)
    assert_would_change(case, exp, where=[i for i, s in enumerate(rec["rank_slot"]) if s == qb])
    check([case], select(frame_of([case]), [case]))


def heavy_value_case(dt, p, seed, tiles=3):
    """One value fills 99.5 % of every tile; it lies under target prefix A, whose cell at pass p B shares, and B's values
    (the linear search) are spread among its rows.  Ranks: the ends of the run, its neighbours, and B."""
    rng = np.random.default_rng(seed)
    n = TILE_MIN * tiles
    decided = pass_geometry(KEY_BITS[dt])[p][2]
    a, b = colliding_cell(dt, decided, rng, need=2)[:2]
    side = block(dt, a, decided, 40, rng)
    heavy = np.sort(side)[20]
    side = side[side != heavy]
    bs = block(dt, b, decided, 60, rng)
    keys = np.full(n, heavy, U64)
    rows = rng.choice(n, side.size + bs.size, replace=False)
    keys[rows] = np.concatenate([side, bs])
    valid = np.ones(n, bool)
    valid[rng.choice(np.setdiff1d(np.arange(n), rows), 30, replace=False)] = False
    srt = np.sort(keys[valid])
    lo, hi = int(np.searchsorted(srt, heavy, "left")), int(np.searchsorted(srt, heavy, "right"))
    ranks = [lo, lo + 1, hi, hi + 1, (lo + hi) // 2] + _ranks_in(srt, b, decided, (0.1, 0.6))
    return Case("run_%s_pass%d" % (dt, p), dt, keys, valid, ranks, p=p, decided=decided, a=a, b=b, heavy=heavy)


@pytest.mark.parametrize("dt,p", TAIL, ids=["%s-pass%d" % a for a in TAIL])
def test_one_value_filling_the_tiles_next_to_a_colliding_prefix(dt, p):
    case = heavy_value_case(dt, p, seed=900 + TAIL.index((dt, p)))
    tr = tile_rows(case.keys.size, 1, _sms())
    per_tile = (case.keys == case.info["heavy"]).reshape(-1, tr).mean(axis=1)
    assert per_tile.size >= 3 and (per_tile > 0.99).all()
    exp = case.expected()
    got_r, passes = case.replay()
    assert _same_float(got_r, exp)
    rec, qa, qb = assert_collision(case, passes)
    assert rec["counted"][qa] > 0.99 * case.keys.size
    assert_would_change(case, exp, where=[i for i, s in enumerate(rec["rank_slot"]) if s == qb])
    check([case], select(frame_of([case]), [case]))


# ---- 6: the per-partition protocol -------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def suite_cases(collision_cases):
    """The columns of items 2 to 4, one frame."""
    small = [collision_case(dt, p, seed=1000 + 10 * i, n_a=600, n_b=1800, n_f=800, n_bg=4000, null_rows=600)
             for i, (dt, p) in enumerate(ALL_PASSES)]
    return (small + [foreign_heavy_case("f64", 4, 1200), foreign_heavy_case("i32", 2, 1201)]
            + [sixteen_slots_case(dt, 1300 + i) for i, dt in enumerate(("f32", "i64"))]
            + [one_slot_case(dt, 1400 + i) for i, dt in enumerate(("i32", "f64"))]
            + [edge_ranks_case(dt, 1500 + i) for i, dt in enumerate(("f32", "i64"))]
            + forty_ranks_cases()[:2])


def _loser_rows(c):
    """Rows holding the prefix that takes the linear search at the case's pass (none for cases without one)."""
    if "b" not in c.info:
        return np.zeros(c.keys.size, bool)
    return in_prefix(c.keys, c.info["b"], c.info["decided"])


def uneven_chunks(cases, n, rng):
    """Chunks of 0, 1, 33 and 4 097 rows, then one that alone holds every column's colliding prefix B, then 777 rows
    null in every column (B-prefix values underneath), then two uneven pieces.  Each column's rows are reordered so
    that its B rows fall in that chunk (the order statistics do not depend on row order)."""
    from anovos_b200.frame import ColumnFrame, _pack_validity
    head = 1 + 33 + 4097
    nb = max(int(_loser_rows(c).sum()) for c in cases)
    cols = {}
    for c in cases:
        vals, valid = np.concatenate([c.vals, np.resize(c.vals, n - c.keys.size)]), \
            np.concatenate([c.valid, np.zeros(n - c.keys.size, bool)])
        lose = np.concatenate([_loser_rows(c), np.zeros(n - c.keys.size, bool)])
        other = rng.permutation(np.flatnonzero(~lose))
        k = nb - int(lose.sum())
        order = np.concatenate([other[:head], np.flatnonzero(lose), other[head:head + k], other[head + k:]])
        vals, valid = vals[order], valid[order]
        under = vals[np.flatnonzero(lose)[:1]] if lose.any() else vals[:1]
        vals = np.concatenate([vals[:head + nb], np.resize(under, 777), vals[head + nb:]])
        valid = np.concatenate([valid[:head + nb], np.zeros(777, bool), valid[head + nb:]])
        cols[c.name] = (vals, valid)
    total = n + 777
    rest = total - head - nb - 777
    bounds = np.cumsum([0, 0, 1, 33, 4097, nb, 777, rest // 3, rest - rest // 3])
    frames = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        data = {}
        for name, (vals, valid) in cols.items():
            v = valid[lo:hi]
            data[name] = (np.ascontiguousarray(vals[lo:hi]), None if v.all() else _pack_validity(v))
        frames.append(ColumnFrame.from_tensors(data, n_rows=int(hi - lo)))
    whole = ColumnFrame.from_tensors({k: (v, _pack_validity(m)) for k, (v, m) in cols.items()}, n_rows=total)
    return frames, whole, bounds, cols


@pytest.mark.parametrize("how", ["rows32", "rows4128", "uneven"])
def test_partitioned_equals_resident(how, suite_cases):
    from anovos_b200.partitioned import PartitionedFrame
    cases = suite_cases
    n = max(c.keys.size for c in cases)
    rk = rank_matrix(cases)
    assert rk.shape[1] > SEL_MAX_RANKS
    fr = frame_of(cases, n)
    for c in fr.columns:
        fr.column(c).device()
    if how == "uneven":
        frames, fr, bounds, cols = uneven_chunks(cases, n, np.random.default_rng(1600))
        assert np.diff(bounds)[0] == 0 and np.diff(bounds)[5] == 777
        for c in cases:
            vals, valid = cols[c.name]
            assert not valid[bounds[5]:bounds[6]].any()                  # the all-null chunk
            if "b" in c.info:                                           # B's valid values only in chunk 4
                rows = np.flatnonzero(in_prefix(sort_key(vals, c.dt), c.info["b"], c.info["decided"]) & valid)
                assert rows.size and rows.min() >= bounds[4] and rows.max() < bounds[5], c.name
        part = PartitionedFrame.from_frames(frames)
    else:
        part = PartitionedFrame.from_frame(fr, int(how[4:]))
        assert part.n_chunks == -(-n // int(how[4:]))
    resident = select(fr, cases, rk)
    got = select(part, cases, rk)
    assert np.array_equal(got.view(U64), resident.view(U64))
    check(cases, got)


# ---- 7: a public function on collision columns -----------------------------------------------------------------------

def percentile_case(dt, p, seed, n=60_000):
    """Summary percentiles 1 .. 25 % in prefix A, 50 .. 99 % in B, one cell at pass p: the ascending ranks give A the
    first slot, B (70 % of the values) takes the linear search.  Values of magnitude >= 1, so that the four decimals of
    the table tell the selected values apart."""
    from anovos_b200 import engine
    from anovos_b200.profile import SUMMARY_PROBS
    from anovos_b200.shared.gk import SUMMARY_EPS
    rng = np.random.default_rng(seed)
    decided = pass_geometry(KEY_BITS[dt])[p][2]
    def shown(q):                                        # every value of the prefix is at least 1 in magnitude
        ends = key_value(np.array([q, q + 1], U64) << U64(64 - decided), dt).astype(np.float64)
        return dt == "i64" or (np.abs(ends) >= 1).all()
    a, b = next(c for c in (colliding_cell(dt, decided, rng, need=2) for _ in range(100)) if shown(c[0]) and shown(c[1]))[:2]
    keys = np.concatenate([block(dt, a, decided, int(0.3 * n), rng), block(dt, b, decided, n - int(0.3 * n), rng)])
    valid = np.ones(n, bool)
    keys, valid = _shuffle(rng, keys, valid)
    ranks = sorted(set(engine.quantile_ranks(n, SUMMARY_PROBS, SUMMARY_EPS)))
    return Case("pct_%s_pass%d" % (dt, p), dt, keys, valid, ranks, p=p, decided=decided, a=a, b=b)


def test_percentiles_of_collision_columns(monkeypatch):
    import pyarrow as pa
    import anovos.data_analyzer.stats_generator as sg
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    from oracle import api as O
    cases = [percentile_case("f64", 2, 1700), percentile_case("f64", 3, 1701), percentile_case("i64", 2, 1702),
             percentile_case("i64", 4, 1703)]
    for c in cases:
        rec, qa, qb = assert_collision(c, c.replay()[1])
        assert all(s == qb for s in rec["rank_slot"][4:]) and rec["counted"][qb] > rec["counted"][qa]
        assert_would_change(c, c.expected(), ("drop",), where=range(4, 9))
    t = pa.table({c.name: pa.array(c.vals) for c in cases})
    seen = []
    real = engine.select_ranks
    monkeypatch.setattr(engine, "select_ranks", lambda fr, names, rk: seen.extend(names) or real(fr, names, rk))
    got = sg.measures_of_percentiles(None, ColumnFrame.from_arrow(t)).toPandas()
    exp = O.measures_of_percentiles(t)
    assert sorted(seen) == sorted(t.column_names)
    cols = ["min", "1%", "5%", "10%", "25%", "50%", "75%", "90%", "95%", "99%", "max"]
    assert list(got["attribute"]) == list(exp["attribute"])
    assert np.array_equal(got[cols].values.astype(float), exp[cols].values.astype(float)), (got, exp)
