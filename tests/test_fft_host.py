"""CPU: the exact tier of the scalar-field FFTs (tests/fft_exact.py) against the DFT definition, the reference's PeerDAS cells through
it, and every status of the FFT entries, which are decided before any device work."""
import ctypes
import hashlib
import random

import pytest

import fft_exact as X


@pytest.mark.parametrize("fid", range(4))
def test_transcription_equals_definition(fid):
    fld = X.FIELDS[fid]
    r = fld.modulus
    rnd = random.Random(fid)
    g = rnd.randrange(2, r)
    descs = {}
    for logn in range(7):
        n = 1 << logn
        for order in sorted({n, 4 * n, 1 << 10}):
            k = order.bit_length() - 1
            if order not in descs:
                descs[order] = X.Descriptor(r, order, X.root_of_unity(r, k))
            d = descs[order]
            w = pow(d.roots[1], order // n, r)           # the stride rule: w_n = w^(N / n)
            a = [rnd.randrange(r) for _ in range(n)]
            for kind in X.KINDS:
                st, out = X.ref_fft(d, kind, a, g if kind.startswith("coset") else None)
                assert st == 0
                assert out == X.expected(kind, a, w, r, g), (kind, n, order)


def test_transcription_statuses():
    r = X.FIELDS[1].modulus
    d = X.Descriptor(r, 16, X.root_of_unity(r, 4))
    assert X.ref_fft(d, "fft_nn", [0] * 32)[0] == 2
    assert X.ref_fft(d, "fft_nn", [])[0] == 3
    assert X.ref_fft(d, "fft_nn", [0] * 12)[0] == 3


def test_peerdas_cells_through_the_exact_tier():
    r = X.FIELDS[0].modulus
    d = X.Descriptor(r, 8192, X.peerdas_omega())
    blobs, cases = X.peerdas_fixture()
    assert len(cases) == 7
    for c in cases:
        cells = X.peerdas_cells_via_fft(blobs[c["blob"]], lambda kind, v: X.ref_fft(d, kind, v)[1])
        assert [hashlib.sha256(x).hexdigest() for x in cells] == c["cell_sha256"], c["name"]


@pytest.mark.parametrize("fid", range(4))
def test_oracle_equals_transcription(fid):
    """oracle_fft (tools/fft_oracle.c, threaded C) gives the exact tier's bytes up to 2^12, batch 1 and 3, every kind."""
    import numpy as np
    import fft_oracle as O
    fld = X.FIELDS[fid]
    r = fld.modulus
    k = 13
    w = X.root_of_unity(r, k)
    desc = X.Descriptor(r, 1 << k, w)
    rnd = random.Random(40 + fid)
    g = rnd.randrange(2, r)
    for logn in range(13):
        n = 1 << logn
        for batch in (1, 3):
            vals = [rnd.randrange(r) for _ in range(n * batch)]
            a = np.frombuffer(X.to_bytes(vals), dtype=np.uint64).reshape(-1, 4)
            for kind in X.KINDS:
                gg = g if kind.startswith("coset") else None
                st, out = O.fft(fld, kind, a, n, X.mont_struct(fld, w), k, X.mont_struct(fld, g) if gg else None)
                want = []
                for b in range(batch):
                    want += X.ref_fft(desc, kind, vals[b * n:(b + 1) * n], gg)[1]
                assert st == 0 and X.from_bytes(out.tobytes()) == want, (kind, n, batch)
    st, _ = O.fft(fld, "fft_nn", np.zeros((12, 4), np.uint64), 12, X.mont_struct(fld, w), k)
    assert st == 3
    st, _ = O.fft(fld, "fft_nn", np.zeros((1 << 14, 4), np.uint64), 1 << 14, X.mont_struct(fld, w), k)
    assert st == 2
    a = np.frombuffer(X.to_bytes([rnd.randrange(r) for _ in range(100)]), dtype=np.uint64).reshape(-1, 4)
    xs = X.from_bytes(a.tobytes())
    assert int.from_bytes(O.evaluate(fld, a, X.mont_struct(fld, 9)), "little") == sum(c * pow(9, j, r) for j, c in enumerate(xs)) % r


# ---- statuses, before any device work -----------------------------------------------------------------------------------
def _lib():
    from constantine_b200 import _lib
    return _lib.load()


def _omega_struct(fid, k):
    fld = X.FIELDS[fid]
    return X.mont_struct(fld, X.root_of_unity(fld.modulus, k))


def _domain_new(fid, omega, k):
    st = ctypes.c_int(-1)
    h = _lib().ctt_b200_fft_domain_new(fid, omega, k, ctypes.byref(st))
    return h, st.value


def test_domain_statuses():
    for fid in range(4):
        fld = X.FIELDS[fid]
        k = 6
        w = X.root_of_unity(fld.modulus, k)
        assert _domain_new(fid, X.mont_struct(fld, w * w % fld.modulus), k) == (None, 4)       # order 2^(k-1)
        assert _domain_new(fid, X.mont_struct(fld, w), k + 1) == (None, 4)                    # order 2^k < 2^(k+1)
        assert _domain_new(fid, X.mont_struct(fld, 5), k) == (None, 4)
        assert _domain_new(fid, X.mont_struct(fld, 5), 0) == (None, 4)
        assert _domain_new(fid, X.mont_struct(fld, fld.modulus - 1), 2) == (None, 4)         # -1 has order 2
        adic = min(X.two_adicity(fld.modulus), 28)
        assert _domain_new(fid, _omega_struct(fid, 4), adic + 1) == (None, 2)
        assert _domain_new(fid, None, 4) == (None, 5)
        assert _domain_new(fid, _omega_struct(fid, 4), -1) == (None, 5)
    assert _domain_new(1, _omega_struct(1, 28), 29) == (None, 2)                               # BN254: 2-adicity 28
    assert _domain_new(0, _omega_struct(0, 28), 29) == (None, 2)                               # above 28
    for bad in (-1, 4, 5):
        assert _domain_new(bad, _omega_struct(0, 4), 4) == (None, 5)


def test_call_statuses_leave_outputs_untouched():
    lib = _lib()
    fld = X.FIELDS[2]
    h, st = _domain_new(2, _omega_struct(2, 4), 4)
    assert st == 0 and h
    try:
        rnd = random.Random(5)
        vals = X.to_bytes([rnd.randrange(fld.modulus) for _ in range(32)])
        src = ctypes.create_string_buffer(vals, len(vals))
        sentinel = bytes([0xA5]) * len(vals)
        out = ctypes.create_string_buffer(sentinel, len(vals))
        g = ctypes.create_string_buffer(X.mont_struct(fld, 3), 32)
        zero = ctypes.create_string_buffer(32)
        for entry in (lib.ctt_b200_fft, lib.ctt_b200_fft_device):
            for kind in range(8):
                sh = g if kind >= 4 else None
                assert entry(h, kind, out, src, 32, 1, sh) == 2            # n > N
                assert entry(h, kind, out, src, 0, 1, sh) == 3
                assert entry(h, kind, out, src, 12, 1, sh) == 3
                assert entry(h, kind, out, src, 32, 0, sh) == 2            # the length comes first
                assert entry(h, kind, None, src, 16, 1, sh) == 5
                assert entry(h, kind, out, None, 16, 1, sh) == 5
                assert entry(None, kind, out, src, 16, 1, sh) == 5
                assert entry(h, kind, out, src, 16, 1 << 62, sh) == 5      # n * batch overflows
            for kind in range(4, 8):
                assert entry(h, kind, out, src, 16, 1, None) == 5
                assert entry(h, kind, out, src, 16, 1, zero) == 5
            assert entry(h, 8, out, src, 16, 1, None) == 5
            assert entry(h, -1, out, src, 16, 1, None) == 5
        assert out.raw == sentinel
    finally:
        lib.ctt_b200_fft_domain_free(h)


def test_python_domain_errors():
    from constantine_b200 import msm as M
    with pytest.raises(M.FFTError) as e:
        M.FFTDomain("bn254_snarks", _omega_struct(1, 3), 4)
    assert e.value.status == 4
    with pytest.raises(M.FFTError) as e:
        M.FFTDomain(7, _omega_struct(1, 3), 3)
    assert e.value.status == 5
    d = M.FFTDomain("vesta", _omega_struct(3, 3), 3)
    try:
        with pytest.raises(M.FFTError) as e:
            d.fft_nn(bytes(32 * 16))
        assert e.value.status == 2
        with pytest.raises(M.FFTError) as e:
            d.coset_ifft_rn(bytes(32 * 4), bytes(32))
        assert e.value.status == 5
    finally:
        d.free()
