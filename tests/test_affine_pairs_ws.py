"""GPU (-m gpu): the warp-specialised batched-affine pair kernel (k_affine_pairs_ws, msm_affine.cuh) at sizes where every consumer
warp walks its shared-memory ring many times over (hundreds of slots per thread at N = 2^20), against closed forms.
Points are k_i * G, so the MSM is (sum k_i s_i) * G."""
import numpy as np
import pytest

from helpers import CURVES, pyref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=[("bls12_381_g1", 20), ("bn254_snarks_g1", 18)], ids=lambda p: "%s-2^%d" % p)
def case(request):
    import torch
    from constantine_b200 import _lib
    curve, logn = request.param
    lib = _lib.load()
    cv = CURVES[curve]
    n = 1 << logn
    rng = np.random.default_rng(logn)
    k = rng.integers(1, 2**63, size=n, dtype=np.uint64)
    gen = b"".join(cv.fp.to_mont(c).to_bytes(cv.fp.nbytes, "little") for coord in cv.gen for c in coord)
    pts = np.empty((n, cv.aff_bytes), dtype=np.uint8)
    assert lib.ctt_b200_scalar_mul_u64(cv.curve_id, gen, k.ctypes.data, n, pts.ctypes.data) == 0
    s = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    s[:, 31] &= 0x1F
    e = sum(int(x) * int.from_bytes(s[i].tobytes(), "little") for i, x in enumerate(k)) % cv.fr.modulus
    want = pyref.ec_mul_fast(e, cv.gen, cv)
    return cv, n, pts, s, torch.from_numpy(pts).cuda(), torch.from_numpy(s).cuda(), want


@pytest.mark.parametrize("levels", [1, 2, 3, 4])
def test_forced_levels_device_resident(case, levels):
    from constantine_b200 import _lib, msm as M
    cv, n, _, _, d_pts, d_s, want = case
    lib = _lib.load()
    try:
        lib.ctt_b200_set_affine_levels(levels)
        got = M.msm_device_ptrs(cv, d_s.data_ptr(), d_pts.data_ptr(), n)
        assert M.last_stats()["affine_levels"] == levels
        assert pyref.jac_bytes_to_affine(got, cv) == want
    finally:
        lib.ctt_b200_set_affine_levels(-1)


@pytest.mark.parametrize("pieces", [2, 4])
def test_point_pieces_host_call(case, pieces):
    """level 0 split by the point pieces of a host call: one launch per piece over a permuted slot list (perm / range)"""
    from constantine_b200 import _lib, msm as M
    cv, n, pts, s, _, _, want = case
    lib = _lib.load()
    tp = M.Threadpool.new(1)
    try:
        lib.ctt_b200_set_point_chunks(pieces)
        for levels in (3, 1):
            lib.ctt_b200_set_affine_levels(levels)
            got = M.multi_scalar_mul_vartime_parallel(tp, cv, s.tobytes(), pts.tobytes(), n)
            assert M.last_stats()["affine_levels"] == levels
            assert pyref.jac_bytes_to_affine(got, cv) == want, (pieces, levels)
    finally:
        lib.ctt_b200_set_point_chunks(0)
        lib.ctt_b200_set_affine_levels(-1)
        tp.shutdown()
