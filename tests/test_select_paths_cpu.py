"""CPU tests of the restatement of the radix select (csrc/select.cu) that test_gpu_select_paths.py builds its columns with:
the constants are the kernel's, the key orders values as NumPy does, the host replay of the passes selects what np.sort
selects, and every collision column of the GPU tests has its collision at the intended pass."""
import os

import numpy as np
import pytest

from test_gpu_select_paths import (ALL_PASSES, CELLS, HASH_HI, HASH_LO, KEY_BITS, NP, SEL_BITS, SEL_BITS0, SEL_MAX_RANKS,
                                   assert_collision, assert_would_change, collision_case, key_value, pass_geometry,
                                   prefix_hash, reference, replay_values, sort_key)

SELECT_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "anovos_b200", "csrc", "select.cu")


def test_restatement_names_the_kernel_constants():
    src = open(SELECT_CU).read()
    assert "0x%08Xu" % HASH_LO in src and "0x%08Xu" % HASH_HI in src
    assert "SEL_BITS0 = %d, SEL_BITS = %d;" % (SEL_BITS0, SEL_BITS) in src
    assert "constexpr int SEL_MAX_RANKS = %d;" % SEL_MAX_RANKS in src
    assert "key_bits == 32 ? %d : (key_bits == 64 ? %d : -1)" % (len(pass_geometry(32)), len(pass_geometry(64))) in src


def test_pass_geometry():
    assert [g[0] for g in pass_geometry(32)] == [12, 10, 10]
    assert [g[0] for g in pass_geometry(64)] == [12, 10, 10, 10, 10, 10, 2]
    for kb in (32, 64):
        for bits, shift, decided in pass_geometry(kb):
            assert shift == 64 - decided - bits and shift >= 64 - kb


def test_prefix_hash_cells():
    """At pass 1 the 4 096 prefixes fill cells of at most two; two prefixes with the same parent (equal but for the low
    10 bits) never share a cell, so from pass 2 on colliding targets always come from different parents."""
    counts = np.bincount(prefix_hash(np.arange(CELLS, dtype=np.uint64)), minlength=CELLS)
    assert counts.max() == 2 and (counts == 2).sum() == 409
    assert prefix_hash(2)[0] == prefix_hash(0xA1A)[0]
    d = (np.arange(1, 1 << SEL_BITS, dtype=np.uint64) * np.uint64(HASH_LO)) & np.uint64(0xFFFFFFFF)
    assert ((d >= 1 << (32 - SEL_BITS0)) & (d <= (1 << 32) - (1 << (32 - SEL_BITS0)))).all()


def _column(dt, n, rng):
    if dt == "f32":
        x = rng.choice(np.concatenate([rng.normal(0, 1e3, 64), [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45]]), n)
    elif dt == "f64":
        x = np.where(rng.random(n) < 0.05, rng.choice([0.0, -0.0, np.nan, -np.inf, 5e-324, 1e300], n), rng.normal(0, 1e6, n))
    elif dt == "i32":
        x = rng.integers(-2 ** 31, 2 ** 31, n)
    else:
        x = np.where(rng.random(n) < 0.5, rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64), rng.integers(-50, 50, n))
    return rng.permutation(np.asarray(x).astype(NP[dt])), rng.random(n) >= 0.1


@pytest.mark.parametrize("dt", ["f32", "i32", "f64", "i64"])
def test_key_orders_like_numpy(dt):
    x, _ = _column(dt, 5000, np.random.default_rng(3))
    k = sort_key(x, dt)
    ref = np.sort(x.astype(np.float64) if dt[0] == "f" else x)
    got = x[np.argsort(k, kind="stable")]
    assert np.array_equal(got.astype(np.float64), ref.astype(np.float64), equal_nan=True)
    back = key_value(k, dt)
    same = (back == x) | (np.isnan(back) & np.isnan(x)) if dt[0] == "f" else back == x
    assert same.all()


@pytest.mark.parametrize("dt", ["f32", "i32", "f64", "i64"])
def test_replay_selects_what_np_sort_selects(dt):
    rng = np.random.default_rng(11 + KEY_BITS[dt])
    for n in (1, 7, 5003):
        x, valid = _column(dt, n, rng)
        valid[0] = True
        nv = int(valid.sum())
        ranks = [0, 1, nv] + list(rng.integers(1, nv + 1, 13))
        got, passes = replay_values(x, valid, ranks, dt)
        assert len(passes) == len(pass_geometry(KEY_BITS[dt]))
        assert np.array_equal(got, reference(x, valid, ranks), equal_nan=True), (dt, n)


@pytest.mark.parametrize("dt,p", ALL_PASSES, ids=["%s-pass%d" % a for a in ALL_PASSES])
def test_collision_columns_collide_at_their_pass(dt, p):
    """The columns of test_gpu_select_paths.py: the replay selects the exact reference, the targets collide at pass p,
    and a slot table without the linear search or without the prefix compare would select other values."""
    case = collision_case(dt, p, seed=100 + 10 * ALL_PASSES.index((dt, p)))
    exp = case.expected()
    got, passes = case.replay()
    assert np.array_equal(got, exp, equal_nan=True)
    rec, qa, qb = assert_collision(case, passes)
    assert_would_change(case, exp, ("drop",), where=[i for i, s in enumerate(rec["rank_slot"]) if s == qb])
    assert_would_change(case, exp, ("cell",))
