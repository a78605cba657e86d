"""GPU (-m gpu): the scalar-field FFTs against the exact tier (tests/fft_exact.py): every field and kind at every length up to 2^14
(the pass switch at 2^12 / 2^13 included), large transforms by closed-form samples and round trips up to BN254's full 2^28 domain,
the stride rule, the reference's PeerDAS cells through both entries, edge inputs, and the device entry's stream and slot contract."""
import ctypes
import hashlib
import random
import threading
import time

import numpy as np
import pytest

import fft_exact as X

pytestmark = pytest.mark.gpu
SPIN_MS = 150


@pytest.fixture(scope="module")
def M():
    from constantine_b200 import msm
    return msm


@pytest.fixture(scope="module")
def lib():
    from constantine_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module", autouse=True)
def engine_defaults(lib):
    import torch
    lib.ctt_b200_set_stream(None)
    lib.ctt_b200_set_concurrency(2)
    try:
        yield
    finally:
        torch.cuda.synchronize()
        lib.ctt_b200_set_stream(None)
        lib.ctt_b200_set_concurrency(2)


def make_domain(M, fid, k):
    fld = X.FIELDS[fid]
    w = X.root_of_unity(fld.modulus, k)
    return M.FFTDomain(fid, X.mont_struct(fld, w), k), w


def rand_vals(r, count, rnd):
    return [rnd.randrange(r) for _ in range(count)]


def expected_batch(desc, kind, vals, n, g=None):
    out = []
    for b in range(len(vals) // n):
        out += X.ref_fft(desc, kind, vals[b * n:(b + 1) * n], g)[1]
    return out


def run(d, kind, vals, batch, gs):
    fn = getattr(d, kind)
    b = X.to_bytes(vals)
    return X.from_bytes(fn(b, gs, batch=batch) if kind.startswith("coset") else fn(b, batch=batch))


@pytest.mark.parametrize("fid", range(4))
def test_every_kind_and_length_exact(M, fid):
    fld = X.FIELDS[fid]
    r = fld.modulus
    rnd = random.Random(100 + fid)
    d, w = make_domain(M, fid, 14)
    desc = X.Descriptor(r, 1 << 14, w)
    g = rnd.randrange(2, r)
    gs = X.mont_struct(fld, g)
    try:
        for logn in range(15):
            n = 1 << logn
            for batch in ((1, 3) if logn <= 12 else (1,)):
                vals = rand_vals(r, n * batch, rnd)
                for kind in X.KINDS:
                    gg = g if kind.startswith("coset") else None
                    assert run(d, kind, vals, batch, gs) == expected_batch(desc, kind, vals, n, gg), (kind, n, batch)
    finally:
        d.free()


def _np_vals(r, count, seed):
    """Random residues as uint64[count, 4], below r (top limb below r's)."""
    rng = np.random.default_rng(seed)
    v = rng.integers(0, 2 ** 64, size=(count, 4), dtype=np.uint64)
    v[:, 3] = rng.integers(0, r >> 192, size=count, dtype=np.uint64)
    return v


@pytest.mark.parametrize("logn", [20, 23, 24, 25])
@pytest.mark.parametrize("fid", [1, 0])
def test_large_every_kind_against_the_oracle(M, fid, logn):
    """Full outputs against the threaded C oracle (tools/fft_oracle.c) at the 2 -> 3 pass switch (2^24 / 2^25) and on both
    sides of it, every kind, one domain of order 2^25 (stride rule included)."""
    import fft_oracle as O
    fld = X.FIELDS[fid]
    r = fld.modulus
    n = 1 << logn
    d, w = make_domain(M, fid, 25)
    omega = X.mont_struct(fld, w)
    gs = X.mont_struct(fld, 5)
    try:
        a = _np_vals(r, n, logn)
        for kind in X.KINDS:
            coset = kind.startswith("coset")
            got = getattr(d, kind)(a, gs) if coset else getattr(d, kind)(a)
            st, want = O.fft(fld, kind, a, n, omega, 25, gs if coset else None)
            assert st == 0 and np.array_equal(got, want), kind
    finally:
        d.free()


def test_bn254_full_domain_2_28(M):
    import torch
    fld = X.FIELDS[1]
    r = fld.modulus
    logn = 28
    n = 1 << logn
    d, w = make_domain(M, 1, logn)
    try:
        g = torch.Generator(device="cuda").manual_seed(28)
        x = torch.randint(-2 ** 63, 2 ** 63 - 1, (n, 4), dtype=torch.int64, device="cuda", generator=g)
        x[:, 3] = torch.randint(0, r >> 192, (n,), dtype=torch.int64, device="cuda", generator=g)
        y = torch.empty_like(x)
        torch.cuda.synchronize()                      # torch's stream is not ordered with the engine's
        d.fft_nn_device(y.data_ptr(), x.data_ptr(), n)
        z = torch.empty_like(x)
        d.ifft_nn_device(z.data_ptr(), y.data_ptr(), n)
        assert torch.equal(x, z)
        del z
        # dense input: 4 sampled outputs, each evaluated in O(n) by the threaded C oracle
        import fft_oracle as O
        xh = x.cpu().numpy().view(np.uint64)
        for k in (1, n - 1, 12345677, 200000003):
            got = y[k].cpu().numpy().tobytes()
            assert got == O.evaluate(fld, xh, X.mont_struct(fld, pow(w, k, r))), k
        del xh
        # 16 non-zero coefficients: 4096 sampled outputs against their closed form
        rnd = random.Random(2828)
        pos = rnd.sample(range(n), 16)
        coef = rand_vals(r, 16, rnd)
        x.zero_()
        x[pos] = torch.tensor(np.frombuffer(X.to_bytes(coef), dtype=np.int64).reshape(16, 4), device="cuda")
        torch.cuda.synchronize()
        d.fft_nn_device(y.data_ptr(), x.data_ptr(), n)
        ks = [0, n - 1] + [rnd.randrange(n) for _ in range(4094)]
        got = y[ks].cpu().numpy()
        for k, row in zip(ks, got):
            want = sum(c * pow(w, (j * k) % n, r) for j, c in zip(pos, coef)) % r
            assert int.from_bytes(row.tobytes(), "little") == want, k
    finally:
        d.free()
        torch.cuda.empty_cache()


def test_stride_rule(M):
    fld = X.FIELDS[0]
    r = fld.modulus
    big, w = make_domain(M, 0, 20)
    small = M.FFTDomain(0, X.mont_struct(fld, pow(w, 1 << 10, r)), 10)
    rnd = random.Random(7)
    gs = X.mont_struct(fld, 11)
    try:
        vals = X.to_bytes(rand_vals(r, 1 << 10, rnd) * 2)
        for kind in X.KINDS:
            args = (vals, gs) if kind.startswith("coset") else (vals,)
            assert getattr(big, kind)(*args, batch=2) == getattr(small, kind)(*args, batch=2), kind
    finally:
        big.free()
        small.free()


def test_peerdas_cells_through_both_entries(M):
    import torch
    fld = X.FIELDS[0]
    d = M.FFTDomain(0, X.mont_struct(fld, X.peerdas_omega()), 13)
    blobs, cases = X.peerdas_fixture()
    to_m = lambda v: X.to_bytes([fld.to_mont(x) for x in v])
    from_m = lambda b: [fld.from_mont(x) for x in X.from_bytes(b)]

    def host(kind, v):
        return from_m(getattr(d, kind)(to_m(v)))

    def device(kind, v):
        t = torch.tensor(np.frombuffer(to_m(v), dtype=np.int64).reshape(-1, 4), device="cuda")
        getattr(d, kind + "_device")(t.data_ptr(), t.data_ptr(), len(v))        # in place
        return from_m(t.cpu().numpy().tobytes())

    try:
        for c in cases:
            for fft in (host, device):
                cells = X.peerdas_cells_via_fft(blobs[c["blob"]], fft)
                assert [hashlib.sha256(x).hexdigest() for x in cells] == c["cell_sha256"], (c["name"], fft.__name__)
    finally:
        d.free()


@pytest.mark.parametrize("fid", [1, 2])
def test_edge_inputs(M, fid):
    fld = X.FIELDS[fid]
    r = fld.modulus
    d, w = make_domain(M, fid, 13)
    desc = X.Descriptor(r, 1 << 13, w)
    try:
        for n in (1 << 5, 1 << 13):
            inputs = [[0] * n, [r - 1] * n, [7] * n] + [[1 if i == k else 0 for i in range(n)] for k in (0, 1, n - 1)]
            for vals in inputs:
                for kind in X.KINDS:
                    for g in ((r - 1, 3) if kind.startswith("coset") else (None,)):
                        gs = X.mont_struct(fld, g) if g is not None else None
                        assert run(d, kind, vals, 1, gs) == X.ref_fft(desc, kind, vals, g)[1], (kind, n, g)
    finally:
        d.free()


def _tensor(vals):
    import torch
    return torch.tensor(np.frombuffer(X.to_bytes(vals), dtype=np.int64).reshape(-1, 4), device="cuda")


def _vals(t):
    return X.from_bytes(t.cpu().numpy().tobytes())


@pytest.mark.parametrize("logn,batch", [(8, 5), (14, 2)])
def test_device_entry_in_and_out_of_place(M, logn, batch):
    import torch
    fld = X.FIELDS[3]
    r = fld.modulus
    n = 1 << logn
    d, w = make_domain(M, 3, 14)
    rnd = random.Random(logn)
    gs = X.mont_struct(fld, 9)
    try:
        vals = rand_vals(r, n * batch, rnd)
        for kind in X.KINDS:
            want = run(d, kind, vals, batch, gs)
            fn = getattr(d, kind + "_device")
            extra = (gs,) if kind.startswith("coset") else ()
            x = _tensor(vals)
            y = torch.full_like(x, -0x5A5A5A5A5A5A5A5B)
            torch.cuda.synchronize()
            fn(y.data_ptr(), x.data_ptr(), n, *extra, batch=batch)
            assert _vals(y) == want and _vals(x) == vals, kind
            fn(x.data_ptr(), x.data_ptr(), n, *extra, batch=batch)
            assert _vals(x) == want, kind
            t = M.FFTDomain.last_timing()
            assert t["ms_kernels"] > 0 and t["ms_h2d"] == 0
    finally:
        d.free()


@pytest.fixture(scope="module")
def spin():
    import torch
    s = torch.cuda.Stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(cycles):
        with torch.cuda.stream(s):
            a.record()
            torch.cuda._sleep(cycles)
            b.record()
        b.synchronize()
        return a.elapsed_time(b)

    timed(1000)
    probe = 20_000_000
    cycles = int(probe * SPIN_MS / timed(probe))
    assert 100 <= timed(cycles) <= 300

    def go(stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(cycles)
    return go


@pytest.mark.parametrize("hold_slot0", [False, True])
@pytest.mark.parametrize("kind,logn", [("fft_nn", 14), ("ifft_rn", 10), ("coset_fft_nr", 14)])
def test_caller_stream_contract(M, lib, spin, kind, logn, hold_slot0):
    """Input written on the caller's stream behind a spin, the call, the output read on that stream with no synchronisation; with
    slot 0 held by a blocking call on that stream, the call runs on another slot."""
    import torch
    fld = X.FIELDS[1]
    r = fld.modulus
    n = 1 << logn
    d, w = make_domain(M, 1, 14)
    other, _ = make_domain(M, 2, 10)
    gs = X.mont_struct(fld, 6)
    rnd = random.Random(logn)
    vals = rand_vals(r, 2 * n, rnd)
    want = run(d, kind, vals, 2, gs)
    S = torch.cuda.Stream()
    src = torch.tensor(np.frombuffer(X.to_bytes(vals), dtype=np.int64).reshape(-1, 4)).pin_memory()
    x = torch.zeros_like(src, device="cuda")
    y = torch.full_like(x, -0x5A5A5A5A5A5A5A5B)
    torch.cuda.synchronize()
    lib.ctt_b200_set_concurrency(2)
    lib.ctt_b200_set_stream(ctypes.c_void_p(S.cuda_stream))
    holder = None
    try:
        spin(S)
        with torch.cuda.stream(S):
            x.copy_(src, non_blocking=True)
        if hold_slot0:
            small = X.to_bytes(rand_vals(X.FIELDS[2].modulus, 1024, rnd))
            holder = threading.Thread(target=lambda: other.fft_nn(small))
            holder.start()
            time.sleep(0.03)
        extra = (gs,) if kind.startswith("coset") else ()
        getattr(d, kind + "_device")(y.data_ptr(), x.data_ptr(), n, *extra, batch=2)
        with torch.cuda.stream(S):
            got = y.to("cpu", non_blocking=False)
        assert X.from_bytes(got.numpy().tobytes()) == want
    finally:
        if holder:
            holder.join()
        torch.cuda.synchronize()
        lib.ctt_b200_set_stream(None)
        d.free()
        other.free()


@pytest.mark.parametrize("slots", [1, 4])
def test_concurrent_callers(M, lib, slots):
    """8 threads, each on its own field and domain, alternate host and device calls; each checks its own results and timing."""
    import torch
    lib.ctt_b200_set_concurrency(slots)
    jobs = []
    for t in range(8):
        fid, logn = t % 4, (6, 13, 10, 12)[t % 4]
        fld = X.FIELDS[fid]
        rnd = random.Random(1000 + t)
        d, w = make_domain(M, fid, 14 - (t & 1))
        kind = X.KINDS[t]
        g = rnd.randrange(2, fld.modulus)
        vals = rand_vals(fld.modulus, 2 << logn, rnd)
        desc = X.Descriptor(fld.modulus, 1 << (14 - (t & 1)), w)
        jobs.append((d, kind, logn, vals, X.mont_struct(fld, g), expected_batch(desc, kind, vals, 1 << logn, g)))
    errors = []

    def worker(job):
        d, kind, logn, vals, gs, want = job
        try:
            x = _tensor(vals)
            y = torch.empty_like(x)
            extra = (gs,) if kind.startswith("coset") else ()
            for _ in range(3):
                if run(d, kind, vals, 2, gs) != want:
                    errors.append(("host", kind))
                if M.FFTDomain.last_timing()["ms_d2h"] <= 0:
                    errors.append(("timing", kind))
                getattr(d, kind + "_device")(y.data_ptr(), x.data_ptr(), 1 << logn, *extra, batch=2)
                if _vals(y) != want:
                    errors.append(("device", kind))
        except Exception as e:  # noqa: BLE001 -- reported below
            errors.append(repr(e))

    threads = [threading.Thread(target=worker, args=(j,)) for j in jobs]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        lib.ctt_b200_set_concurrency(2)
        for j in jobs:
            j[0].free()
    assert errors == []
