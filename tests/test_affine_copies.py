"""GPU (-m gpu): the copy lists of the batched-affine levels (msm_affine.cuh). At every level a bucket whose count is odd has one
single slot, which is copied outside the pair kernels' shared inversion; these tests design the bucket sizes so that the copies land
at chosen levels: all odd, all even, runs of 1, 2, 3, 2^L - 1, 2^L and 2^L + 1, one run of every entry, and singles whose point is
infinity or carries a negative digit. Points are k_i * G (k_i = 0 for infinity), so the MSM is (sum k_i s_i) * G."""
import numpy as np
import pytest

from helpers import CURVES, pyref

pytestmark = pytest.mark.gpu

RUNS = [1, 2, 3] + [x for L in range(2, 6) for x in ((1 << L) - 1, 1 << L, (1 << L) + 1)]


def design(name, c):
    """(scalars, infinity flags) in sorted-entry order per bucket. A scalar d < 2^(c-1) is the digit d of window 0 only; 2^c - d is
    the digit -d there (the bucket of d, sign bit set) and a carry of 1 into window 1. Digits stay below 32: any c >= 6."""
    neg = lambda d: (1 << c) - d                                     # noqa: E731
    scal, inf = [], []

    def bucket(scalar, size, last_inf=False):
        scal.extend([scalar] * size)
        inf.extend([False] * (size - 1) + [last_inf])

    if name == "all_odd":
        for d in range(1, 32):
            bucket(d, 2 * (d % 9) + 1)
    elif name == "all_even":
        for d in range(1, 32):
            bucket(d, 2 * (d % 9) + 2)
    elif name == "runs":                              # digits 1..15 positive, 17..31 negative: one bucket per run
        for d, size in enumerate(RUNS, start=1):
            bucket(d, size)
            bucket(neg(d + 16), size)
    elif name == "one_run":
        bucket(5, 1000)
    elif name == "inf_and_neg_singles":               # odd runs: their last entry is the single slot of level 0
        odd = [x for x in RUNS if x & 1]
        for d, size in enumerate(odd, start=1):
            bucket(d, size, last_inf=True)            # a single whose point is infinity
            bucket(neg(d + 10), size)                 # a single with the sign bit
            bucket(neg(d + 20), size, last_inf=True)  # both
    return scal, inf


def make_case(lib, cv, name, c, rng):
    scal, inf = design(name, c)
    n = len(scal)
    # stable sort: entries of a bucket keep their index order, so the last one of a run is the highest index
    k = rng.integers(1, 2**63, size=n, dtype=np.uint64)
    gen = b"".join(cv.fp.to_mont(x).to_bytes(cv.fp.nbytes, "little") for coord in cv.gen for x in coord)
    pts = np.empty((n, cv.aff_bytes), dtype=np.uint8)
    assert lib.ctt_b200_scalar_mul_u64(cv.curve_id, gen, k.ctypes.data, n, pts.ctypes.data) == 0
    inf_bytes = np.frombuffer(pyref.aff_to_bytes(None, cv), dtype=np.uint8)
    for i in np.flatnonzero(inf):
        pts[i] = inf_bytes
    s = np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in scal), dtype=np.uint8).reshape(n, 32).copy()
    e = sum(int(x) * v for x, v, z in zip(k, scal, inf) if not z) % cv.fr.modulus
    return n, pts, s, pyref.ec_mul_fast(e, cv.gen, cv)


DESIGNS = ["all_odd", "all_even", "runs", "one_run", "inf_and_neg_singles"]


@pytest.mark.parametrize("levels", [1, 2, 3, 4])
@pytest.mark.parametrize("name", DESIGNS)
@pytest.mark.parametrize("curve", ["bls12_381_g1", "bn254_snarks_g1"])
def test_designed_buckets_device_resident(curve, name, levels):
    import torch
    from constantine_b200 import _lib, msm as M
    lib = _lib.load()
    cv = CURVES[curve]
    c = 10
    n, pts, s, want = make_case(lib, cv, name, c, np.random.default_rng(levels))
    d_pts, d_s = torch.from_numpy(pts).cuda(), torch.from_numpy(s).cuda()
    try:
        lib.ctt_b200_set_affine_levels(levels)
        got = M.msm_device_ptrs(cv, d_s.data_ptr(), d_pts.data_ptr(), n, force_c=c)
        assert M.last_stats()["affine_levels"] == levels
        assert pyref.jac_bytes_to_affine(got, cv) == want, (curve, name, levels)
    finally:
        lib.ctt_b200_set_affine_levels(-1)


@pytest.mark.parametrize("name", ["runs", "inf_and_neg_singles"])
def test_designed_buckets_g2(name):
    """Fp2 coordinates: the copies in k_affine_pairs"""
    import torch
    from constantine_b200 import _lib, msm as M
    lib = _lib.load()
    cv = CURVES["bls12_381_g2"]
    c = 10
    n, pts, s, want = make_case(lib, cv, name, c, np.random.default_rng(2))
    d_pts, d_s = torch.from_numpy(pts).cuda(), torch.from_numpy(s).cuda()
    try:
        for levels in (1, 3):
            lib.ctt_b200_set_affine_levels(levels)
            got = M.msm_device_ptrs(cv, d_s.data_ptr(), d_pts.data_ptr(), n, force_c=c)
            assert M.last_stats()["affine_levels"] == levels
            assert pyref.jac_bytes_to_affine(got, cv) == want, (name, levels)
    finally:
        lib.ctt_b200_set_affine_levels(-1)


@pytest.mark.parametrize("pieces", [2, 4])
@pytest.mark.parametrize("curve", ["bls12_381_g1", "bn254_snarks_g1"])
def test_designed_buckets_point_pieces(curve, pieces):
    """a host call whose points arrive in pieces: level 0's pairs run per piece, its copies in the last launch"""
    from constantine_b200 import _lib, msm as M
    lib = _lib.load()
    cv = CURVES[curve]
    tp = M.Threadpool.new(1)
    try:
        lib.ctt_b200_set_point_chunks(pieces)
        for name in ("runs", "inf_and_neg_singles"):
            c = M.plan(cv, len(design(name, 6)[0]))[0]      # the sizes do not depend on c; the engine's choice decides the digits
            assert c >= 6
            n, pts, s, want = make_case(lib, cv, name, c, np.random.default_rng(pieces))
            for levels in (3, 1):
                lib.ctt_b200_set_affine_levels(levels)
                got = M.multi_scalar_mul_vartime_parallel(tp, cv, s.tobytes(), pts.tobytes(), n)
                assert M.last_stats()["affine_levels"] == levels
                assert pyref.jac_bytes_to_affine(got, cv) == want, (name, pieces, levels)
    finally:
        lib.ctt_b200_set_point_chunks(0)
        lib.ctt_b200_set_affine_levels(-1)
        tp.shutdown()
