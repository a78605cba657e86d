"""EIP-2537 BLS12_G1MSM / BLS12_G2MSM results on the GPU, byte for byte against the model of tests/eip2537_exact.py or its closed
form: scalars at every reduction edge up to 2^256, infinity and cancellations, canonical outputs, every window size the engine
picks for calls of up to 8192 (G1) / 4096 (G2) pairs, random points against the model and the C oracle, and concurrent callers.

Closed forms: the points are built by running sums over bases [b_j]G, so every point is [e_i]G with e_i known, and a call's result
is the one scalar multiplication [sum_i s_i e_i mod r]G."""
import random
import threading

import pytest

import eip2537_exact as E
from test_msm_regimes import plain_regime

GROUPS = {"G1": E.G1, "G2": E.G2}
CURVE = {"G1": "bls12_381_g1", "G2": "bls12_381_g2"}
R = E.R
SIZES_G1 = [1, 2, 3, 4, 7, 8, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 1000, 1024, 2047, 2048,
            4095, 4096, 8191, 8192]
SIZES = {"G1": SIZES_G1, "G2": [k for k in SIZES_G1 if k <= 4096]}


def edge_scalars(rnd):
    """0, 1, 2, r - 1, r, r + 1, 2r - 1, 2r, 2r + 1, 2^255, 2^256 - 1, and random values below r, in [r, 2r) and in [2r, 2^256)"""
    out = [0, 1, 2, R - 1, R, R + 1, 2 * R - 1, 2 * R, 2 * R + 1, 1 << 255, (1 << 256) - 1]
    for _ in range(2):
        out += [rnd.randrange(R), rnd.randrange(R, 2 * R), rnd.randrange(2 * R, 1 << 256)]
    return out


@pytest.fixture(scope="module")
def M():
    from constantine_b200 import msm
    return msm


def call(M, name, inputs):
    fn = M.eth_evm_bls12381_g1msm if name == "G1" else M.eth_evm_bls12381_g2msm
    return fn(inputs)


@pytest.fixture(scope="module")
def pool():
    """per group: 8192 / 4096 points by running sums over four bases [b_j]G, with their discrete logs"""
    rnd = random.Random(197)
    out = {}
    for name, g in GROUPS.items():
        gen = E.generator(g)
        coefs = [rnd.randrange(1, R) for _ in range(4)]
        bases = [E.member(E.ec_mul(c, gen)) for c in coefs]
        out[name] = (gen,) + E.running_sums(bases, coefs, max(SIZES[name]), rnd)
    return out


def closed_form(g, gen, exps, scalars):
    return E.enc_point(g, E.ec_mul(sum(s * e for s, e in zip(scalars, exps)) % R, gen))


# ---------------------------------------------------------------------------------------------------------- CPU: size coverage
def test_sizes_cover_every_engine_plan():
    """The k of the size test reach every (window, batched-affine levels) the engine selects for k <= 8192 (G1) / 4096 (G2)
    pairs, by the mirror of tests/test_msm_regimes.py: a tuning change that moves a threshold fails here."""
    for name, top in (("G1", 8192), ("G2", 4096)):
        every = {plain_regime(CURVE[name], k) for k in range(1, top + 1)}
        assert {plain_regime(CURVE[name], k) for k in SIZES[name]} == every, name
        assert len(every) >= 7


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["G1", "G2"])
def test_scalars_at_every_reduction_edge(M, kat, pool, name):
    """One call of pairs ([a]G, s) and (p1 / p2, s) over the edge scalars, against the model; then each s alone with [a]G."""
    g = GROUPS[name]
    rnd = random.Random(7)
    gen, pts, exps = pool[name]
    base = E.kat_base(kat, g)
    ss = edge_scalars(rnd)
    inputs = b"".join(E.enc_pair(g, pts[i], s) + E.enc_pair(g, base, s) for i, s in enumerate(ss))
    assert call(M, name, inputs) == E.msm(g, inputs)
    for i, s in enumerate(ss):
        got = call(M, name, E.enc_pair(g, pts[i], s))
        assert got == (E.SUCCESS, closed_form(g, gen, [exps[i]], [s])), hex(s)
        got = call(M, name, E.enc_pair(g, base, s))
        assert got == E.msm(g, E.enc_pair(g, base, s)), hex(s)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["G1", "G2"])
def test_infinity_and_cancellation(M, pool, name):
    g = GROUPS[name]
    rnd = random.Random(9)
    gen, pts, exps = pool[name]
    zero = bytes(g.out)
    # the point at infinity with nonzero scalars among finite pairs
    inputs = b"".join(E.enc_pair(g, None if i % 3 == 1 else pts[i], rnd.getrandbits(256)) for i in range(9))
    assert call(M, name, inputs) == E.msm(g, inputs)
    # all-zero scalars
    for k in (1, 5, 300):
        assert call(M, name, b"".join(E.enc_pair(g, p, 0) for p in pts[:k])) == (E.SUCCESS, zero), k
    # (P, s) with (P, r - s) and (P, s) with (-P, s); s alone above 2r
    for i in range(4):
        s = rnd.randrange(1, R)
        assert call(M, name, E.enc_pair(g, pts[i], s) + E.enc_pair(g, pts[i], R - s)) == (E.SUCCESS, zero)
        assert call(M, name, E.enc_pair(g, pts[i], s) + E.enc_pair(g, pts[i], 2 * R - s)) == (E.SUCCESS, zero)
        assert call(M, name, E.enc_pair(g, pts[i], s) + E.enc_pair(g, E.ec_neg(pts[i]), s)) == (E.SUCCESS, zero)
    # k copies of one point: scalars summing to 0 mod r, then random scalars
    for k in (2, 17, 300):
        p, e = pts[k], exps[k]
        ss = [rnd.getrandbits(256) for _ in range(k - 1)]
        last = (-sum(ss)) % R + R * rnd.randrange(2)
        assert call(M, name, b"".join(E.enc_pair(g, p, s) for s in ss + [last])) == (E.SUCCESS, zero), k
        ss.append(rnd.getrandbits(256))
        assert call(M, name, b"".join(E.enc_pair(g, p, s) for s in ss)) == (E.SUCCESS, closed_form(g, gen, [e] * k, ss)), k


def _words(g, out):
    return [int.from_bytes(out[64 * i:64 * i + 64], "big") for i in range(2 * g.degree)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["G1", "G2"])
def test_outputs_are_canonical(M, pool, name):
    """Results R and -R: every output word is below p, x is equal and every word of y sums with its partner to p (or both are 0).
    A subgroup point with a chosen small y cannot be found, so instead every output of 64 pairs of calls is checked this way: a
    conversion out of Montgomery form that skips its final subtraction would leave a word >= p and break the sum."""
    g = GROUPS[name]
    rnd = random.Random(11)
    gen, pts, exps = pool[name]
    for i in range(64):
        s = rnd.randrange(1, R)
        st1, a = call(M, name, E.enc_pair(g, pts[i], s) + E.enc_pair(g, pts[i + 64], rnd.getrandbits(256)) +
                      E.enc_pair(g, pts[i + 64], 0))
        assert st1 == E.SUCCESS
        wa = _words(g, a)
        assert all(a[64 * j:64 * j + 16] == bytes(16) for j in range(2 * g.degree)) and all(w < E.P for w in wa)
        res = E.dec_point(g, a)
        assert res is not None and E.on_curve(g, res)
        st2, b = call(M, name, E.enc_pair(g, E.member(E.ec_neg(res)), 1))   # -R, as the result of a call of its own
        assert st2 == E.SUCCESS
        wb = _words(g, b)
        d = g.degree
        assert wa[:d] == wb[:d]
        assert all((ya + yb == E.P) if ya else yb == 0 for ya, yb in zip(wa[d:], wb[d:]))
        assert all(b[64 * j:64 * j + 16] == bytes(16) for j in range(2 * d))


@pytest.mark.gpu
@pytest.mark.parametrize("name,k", [(n, k) for n in ("G1", "G2") for k in SIZES[n]], ids=str)
def test_sizes_through_engine_plans(M, pool, name, k):
    """k pairs from the pool, salted with infinity pairs, zero scalars and scalars >= 2r, against the closed form; the call ran the
    window size and batched-affine levels the mirror predicts."""
    g = GROUPS[name]
    rnd = random.Random(k)
    gen, pts, exps = pool[name]
    enc, ss, es = [], [], []
    for i in range(k):
        s = rnd.getrandbits(256)
        kind = rnd.randrange(16)
        p, e = pts[i], exps[i]
        if kind == 0:
            p, e = None, 0
        elif kind == 1:
            s = 0
        elif kind == 2:
            s = rnd.randrange(2 * R, 1 << 256)
        enc.append(E.enc_pair(g, p, s))
        ss.append(s)
        es.append(e)
    assert call(M, name, b"".join(enc)) == (E.SUCCESS, closed_form(g, gen, es, ss))
    st = M.last_stats()
    assert (st["c"], st["affine_levels"]) == plain_regime(CURVE[name], k)


def _cleared_points(g, n, rnd):
    """random subgroup points with unknown discrete logs: [h] Q for random curve points Q"""
    return [E.member(E.ec_mul(g.h, E.random_curve_point(g, rnd))) for _ in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["G1", "G2"])
def test_random_points_against_the_model(M, name):
    g = GROUPS[name]
    rnd = random.Random(13)
    qs = _cleared_points(g, 16, rnd)
    for k in (1, 2, 5, 16, 33, 64):
        inputs = b"".join(E.enc_pair(g, qs[rnd.randrange(16)], rnd.getrandbits(256)) for _ in range(k))
        assert call(M, name, inputs) == E.msm(g, inputs), k


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["G1", "G2"])
def test_random_points_against_the_oracle(M, oracle_lib, name):
    """1024 running sums over four random subgroup points, against the C oracle's MSM of the reduced scalars"""
    from helpers import CURVES, pyref
    g = GROUPS[name]
    cv = CURVES[CURVE[name]]
    rnd = random.Random(17)
    bases = _cleared_points(g, 4, rnd)
    cur, pts = [None] * 4, []
    for _ in range(1024):
        j = rnd.randrange(4)
        cur[j] = E.member(E.ec_add(cur[j], bases[j]))
        pts.append(cur[j])
    ss = [rnd.getrandbits(256) for _ in pts]
    st, out = call(M, name, b"".join(E.enc_pair(g, p, s) for p, s in zip(pts, ss)))
    assert st == E.SUCCESS

    def tup(p):
        return None if p is None else tuple(tuple(c[:g.degree]) for c in p)

    cb = b"".join(pyref.scalar_to_bytes(s % R, cv) for s in ss)
    pb = b"".join(pyref.aff_to_bytes(tup(p), cv) for p in pts)
    want = pyref.jac_bytes_to_affine(oracle_lib.msm(cv, cb, pb, len(pts)), cv)
    assert tup(E.dec_point(g, out)) == want


@pytest.mark.gpu
def test_concurrent_callers(M, pool):
    """8 threads, each calling both entries three times on its own inputs; every result equals the serial one"""
    jobs = []
    for t in range(8):
        rnd = random.Random(100 + t)
        job = []
        for name in ("G1", "G2"):
            g = GROUPS[name]
            _, pts, _ = pool[name]
            k = 50 + 37 * t
            job.append((name, b"".join(E.enc_pair(g, pts[rnd.randrange(len(pts))], rnd.getrandbits(256)) for _ in range(k))))
        jobs.append(job)
    serial = [[call(M, name, inp) for name, inp in job] for job in jobs]
    assert all(st == E.SUCCESS for row in serial for st, _ in row)
    results = [None] * 8
    errors = []

    def worker(t):
        try:
            results[t] = [[call(M, name, inp) for name, inp in jobs[t]] for _ in range(3)]
        except Exception as e:   # noqa: BLE001 - reported below
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors
    for t in range(8):
        assert results[t] == [serial[t]] * 3, t
