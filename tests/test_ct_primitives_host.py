"""CPU: the exact model of the secp256k1 folds (tests/secp256k1_fold_exact.py) and the designed inputs that reach their rare steps,
and the call-level checks of the constant-time test hook ctt_b200_test_ct_op (no device work)."""
import ctypes
import random

import pytest

import secp256k1_fold_exact as F
from evm_ecrecover_exact import N, P


@pytest.mark.parametrize("m", ["p", "n"])
def test_fold_model_reduces_random_and_extreme_products(m):
    mod, fold = F.FOLD[m]
    rnd = random.Random(1)
    for T in [0, 1, mod, mod * mod - 1, (mod - 1) ** 2, 2 ** 512 - 1, (2 ** 256 - 1) * mod] + [rnd.getrandbits(512) for _ in range(4000)]:
        r, _ = fold(T)             # the model asserts every bound the device code's comments state, and r = T mod m
        assert r == T % mod


@pytest.mark.parametrize("m", ["p", "n"])
def test_designed_products_take_every_step(m):
    """Every conditional step of the fold, taken and not taken, on canonical pairs (a, b < m). All of them are reachable:
    fold_p's second-stage carry by (2^255, 2H) with H C in [2 2^256 - C, 2^257), fold_n's fourth fold by the pairs whose
    second-stage value lies in [2^257 - C, 2^257), both final subtractions by a b in [m, m + a). Random products do not reach the
    rare ones (fold_p's carry, fold_n's fourth fold, the subtractions), which is why these are built."""
    mod, fold = F.FOLD[m]
    pairs = F.designed_products(mod)
    assert all(0 <= a < mod and 0 <= b < mod for a, b in pairs)
    seen = {s: set() for s in F.STEPS[m]}
    for a, b in pairs:
        _, steps = fold(a * b)
        for s, v in steps.items():
            seen[s].add(v)
    assert all(v == {False, True} for v in seen.values()), seen
    rnd = random.Random(2)
    rare = ("carry", "sub") if m == "p" else ("h4", "sub")
    for _ in range(2000):
        steps = fold(rnd.randrange(mod) * rnd.randrange(mod))[1]
        assert not any(steps[s] for s in rare)


@pytest.mark.parametrize("mod", [P, N], ids=["p", "n"])
def test_designed_sums_and_differences_reach_their_edges(mod):
    sums = {a + b for a, b in F.designed_sums(mod)}
    assert {mod - 1, mod, mod + 1, 2 ** 256 - 1, 2 ** 256, 2 ** 256 + 1, 2 * mod - 2} <= sums
    assert all(a < mod and b < mod for a, b in F.designed_sums(mod) + F.designed_differences(mod))
    diffs = {a - b for a, b in F.designed_differences(mod)}
    assert {-1, 0, 1} <= diffs
    for a, b in F.designed_sums(mod):
        assert F.add_ct(a, b, mod) == (a + b) % mod
    for a, b in F.designed_differences(mod):
        assert F.sub_ct(a, b, mod) == (a - b) % mod


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def test_ct_hook_rejects_unknown_units_ops_and_bad_records():
    lib = _lib()
    buf = ctypes.create_string_buffer(288 * 2)
    known = {0: (0, 1, 2, 8), 1: (0, 1, 2, 8), 2: (0, 2), 3: (8,), 4: (8,), 5: (0, 2), 6: (0, 1, 2)}
    for unit in range(-1, 9):
        for op in range(-1, 16):
            if op in known.get(unit, ()):
                assert lib.ctt_b200_test_ct_op(unit, op, buf, buf, buf, 0) == 0, (unit, op)   # n = 0: no device work
            else:
                assert lib.ctt_b200_test_ct_op(unit, op, buf, buf, buf, 1) == -1, (unit, op)
    # null pointers, and table rows and digits out of range, are refused before any device work
    assert lib.ctt_b200_test_ct_op(0, 0, None, buf, buf, 1) == -1
    assert lib.ctt_b200_test_ct_op(0, 0, buf, buf, None, 1) == -1
    assert lib.ctt_b200_test_ct_op(6, 2, buf, buf, None, 1) == -1
    assert lib.ctt_b200_test_ct_op(2, 0, buf, buf, None, 1) == -1
    assert lib.ctt_b200_test_ct_op(5, 0, buf, buf, None, 1) == -1
    for unit, words, rec in ((2, 24, (64, 1)), (2, 24, (0, 16)), (5, 36, (64, 1)), (5, 36, (63, 16)), (6, 72, (16,))):
        a = (ctypes.c_uint32 * words)(*rec)
        assert lib.ctt_b200_test_ct_op(unit, 2, buf, a, buf, 1) == -1, (unit, rec)
