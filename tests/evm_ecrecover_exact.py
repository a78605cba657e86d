"""Exact model of the ECRECOVER precompile (0x01) as this library computes it (constantine_b200/csrc/evm_secp256k1.cu), written from
the definitions: secp256k1 (SEC 2, section 2.4.1), Keccak-256 (the original Keccak padding, as Ethereum uses) and the reference's
eth_evm_ecrecover (constantine/ethereum_evm_precompiles.nim:1300-1370) with recoverPubkeyImpl_vartime and verifyImpl
(constantine/signatures/ecdsa.nim:258-291, 311-382).

Two forms of the same function:
  - transcribed(): the reference's steps 1-6, including its candidate loop (x1 += n in Fp while x1 <= r), run under an explicit
    iteration cap, with verifyImpl's own conventions (0^-1 = 0, affine (0, 0) is infinity);
  - closed(): the first-candidate rule the device implements: address(Q) for Q = r^-1 (s R - m G) when r, s != 0 (mod n) and r
    lifts, else the zero key (affine (0, 0)), whose address is keccak256(0^64)[12..31].
Plus a cheap builder of many valid signatures (bulk_records) for the large GPU tests.
"""
import random

P = 2 ** 256 - 2 ** 32 - 977
N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
GX = 0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798
GY = 0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8
G = (GX, GY)
B = 7

STATUS = ("cttEVM_Success", "cttEVM_InvalidInputSize", "cttEVM_InvalidOutputSize", "cttEVM_IntLargerThanModulus",
          "cttEVM_PointNotOnCurve", "cttEVM_PointNotInSubgroup", "cttEVM_VerificationFailure", "cttEVM_MalformedSignature")

# ---- Keccak-256 -------------------------------------------------------------------------------------------------------------------
_RC = []
_R = 1
for _ in range(24):
    rc = 0
    for j in range(7):
        # the LFSR x^8 + x^6 + x^5 + x^4 + 1 of FIPS 202, algorithm 5
        if _R & 1:
            rc |= 1 << ((1 << j) - 1)
        _R = ((_R << 1) ^ (0x171 if _R & 0x80 else 0)) & 0xFF
    _RC.append(rc)
_ROT = [[0] * 5 for _ in range(5)]
_x, _y = 1, 0
for _t in range(24):
    _ROT[_x][_y] = ((_t + 1) * (_t + 2) // 2) % 64
    _x, _y = _y, (2 * _x + 3 * _y) % 5
_M64 = (1 << 64) - 1


def _rol(v, n):
    n %= 64
    return ((v << n) | (v >> (64 - n))) & _M64 if n else v


def keccak_f1600(a):
    """a[x][y], 64-bit lanes"""
    for rnd in range(24):
        c = [a[x][0] ^ a[x][1] ^ a[x][2] ^ a[x][3] ^ a[x][4] for x in range(5)]
        d = [c[(x - 1) % 5] ^ _rol(c[(x + 1) % 5], 1) for x in range(5)]
        a = [[a[x][y] ^ d[x] for y in range(5)] for x in range(5)]
        b = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                b[y][(2 * x + 3 * y) % 5] = _rol(a[x][y], _ROT[x][y])
        a = [[b[x][y] ^ (~b[(x + 1) % 5][y] & b[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
        a[0][0] ^= _RC[rnd]
    return a


def keccak256(msg: bytes) -> bytes:
    return sponge256(msg, 0x01)


def sponge256(msg: bytes, pad: int) -> bytes:
    """the rate-136 sponge with a 32-byte output: pad 0x01 is Keccak-256, 0x06 is SHA3-256 (hashlib.sha3_256)"""
    rate = 136
    data = bytearray(msg) + bytes([pad]) + b"\0" * ((-len(msg) - 1) % rate)
    data[-1] |= 0x80
    a = [[0] * 5 for _ in range(5)]
    for off in range(0, len(data), rate):
        block = data[off:off + rate]
        for i in range(rate // 8):
            a[i % 5][i // 5] ^= int.from_bytes(block[8 * i:8 * i + 8], "little")
        a = keccak_f1600(a)
    return b"".join(a[i % 5][i // 5].to_bytes(8, "little") for i in range(4))


# ---- secp256k1 --------------------------------------------------------------------------------------------------------------------
def on_curve(pt):
    return pt is None or (pt[1] * pt[1] - pt[0] ** 3 - B) % P == 0


def _jac_dbl(p):
    x, y, z = p
    if z == 0 or y == 0:
        return (1, 1, 0)
    yy = y * y % P
    s = 4 * x * yy % P
    m = 3 * x * x % P
    x3 = (m * m - 2 * s) % P
    return x3, (m * (s - x3) - 8 * yy * yy) % P, 2 * y * z % P


def _jac_add(p, q):
    if p[2] == 0:
        return q
    if q[2] == 0:
        return p
    z1z1, z2z2 = p[2] * p[2] % P, q[2] * q[2] % P
    u1, u2 = p[0] * z2z2 % P, q[0] * z1z1 % P
    s1, s2 = p[1] * q[2] * z2z2 % P, q[1] * p[2] * z1z1 % P
    h, rr = (u2 - u1) % P, (s2 - s1) % P
    if h == 0:
        return _jac_dbl(p) if rr == 0 else (1, 1, 0)
    hh = h * h % P
    hhh = h * hh % P
    v = u1 * hh % P
    x3 = (rr * rr - hhh - 2 * v) % P
    return x3, (rr * (v - x3) - s1 * hhh) % P, p[2] * q[2] * h % P


def _to_aff(p):
    if p[2] == 0:
        return None
    zi = pow(p[2], -1, P)
    return p[0] * zi * zi % P, p[1] * zi * zi * zi % P


def ec_add(a, b):
    """affine points, None for infinity"""
    ja = (a[0], a[1], 1) if a else (1, 1, 0)
    jb = (b[0], b[1], 1) if b else (1, 1, 0)
    return _to_aff(_jac_add(ja, jb))


def ec_neg(a):
    return None if a is None else (a[0], (-a[1]) % P)


def ec_mul(k, pt):
    if pt is None or k % N == 0:
        return None
    acc, base = (1, 1, 0), (pt[0], pt[1], 1)
    for bit in bin(k % N)[2:]:
        acc = _jac_dbl(acc)
        if bit == "1":
            acc = _jac_add(acc, base)
    return _to_aff(acc)


def ec_lincomb(u1, p1, u2, p2):
    return ec_add(ec_mul(u1, p1), ec_mul(u2, p2))


def sqrt_p(a):
    """a square root of a mod p, or None"""
    y = pow(a, (P + 1) // 4, P)
    return y if y * y % P == a % P else None


def lift_x(x, even):
    """(x, y) on the curve with the requested parity of y, or None"""
    y = sqrt_p((x ** 3 + B) % P)
    if y is None:
        return None
    if (y % 2 == 0) != even:
        y = P - y
    return x, y


def address_of(pt) -> bytes:
    """keccak256(x || y)[12..31]; the affine (0, 0) stands for infinity / no key"""
    x, y = pt if pt is not None else (0, 0)
    return keccak256(x.to_bytes(32, "big") + y.to_bytes(32, "big"))[12:]


ZERO_KEY_ADDRESS = address_of(None)


def record(m, v, r, s):
    """the 128-byte input msg || v || r || s (v an integer, 32 bytes big-endian)"""
    return b"".join(x.to_bytes(32, "big") for x in (m, v, r, s))


def parse(inp):
    """-> (m, v bytes, r, s) as integers (not reduced) and the v word"""
    return (int.from_bytes(inp[0:32], "big"), inp[32:64], int.from_bytes(inp[64:96], "big"), int.from_bytes(inp[96:128], "big"))


def v_check(vw):
    """None when the v word is malformed, else evenY"""
    if any(vw[:31]) or vw[31] not in (0, 1, 27, 28):
        return None
    return vw[31] in (0, 27)


def output_of(addr):
    return b"\0" * 12 + addr


# ---- the reference transcribed ------------------------------------------------------------------------------------------------------
def _inv_n(a):
    return pow(a, -1, N) if a % N else 0          # Fr inv: 0^-1 = 0


def verify_impl(pub, r, s, m):
    """verifyImpl(publicKey, signature, msgHash); pub affine, (0, 0) / None is infinity"""
    if pub == (0, 0):
        pub = None
    w = _inv_n(s)
    u1, u2 = m * w % N, r * w % N
    R = ec_lincomb(u1, G, u2, pub)
    x = R[0] if R is not None else 0              # getAffine of infinity is (0, 0)
    return x % N == r


class CapReached(Exception):
    pass


def recover_transcribed(m, r, s, even, cap):
    """recoverPubkeyImpl_vartime(msgHash = m, signature = (r, s), evenY) with m, r, s already reduced mod n. Returns
    (recovered affine or None for the neutral element, candidates tried, index of the verifying candidate or None). Raises
    CapReached, carrying the same triple, when the loop would run past `cap` candidates."""
    recovered, valid, tried, which = None, False, 0, None
    x1 = r
    while (not valid) and x1 <= r:
        if tried == cap:
            e = CapReached()
            e.state = (recovered, tried, which)
            raise e
        tried += 1
        R = lift_x(x1, even)
        if R is None:
            x1 = (x1 + N) % P
            continue
        r_inv = _inv_n(r)
        u1 = (-(m * r_inv)) % N
        u2 = s * r_inv % N
        Q = ec_lincomb(u1, G, u2, R)
        valid = verify_impl(Q if Q is not None else (0, 0), r, s, m)
        if valid:
            recovered, which = Q, tried - 1
        x1 = (x1 + N) % P
    return recovered, tried, which


def transcribed(inp: bytes, r_len: int = 32, cap: int = 64):
    """eth_evm_ecrecover steps 1-6 -> (status name, 32-byte output or None). r receives only bytes 12..31; the output here is the
    batch form, bytes 0..11 zero. Raises CapReached when the reference's candidate loop exceeds `cap`."""
    if len(inp) != 128:
        return STATUS[1], None
    if r_len != 32:
        return STATUS[2], None
    m, vw, r, s = parse(inp)
    even = v_check(vw)
    if even is None:
        return STATUS[7], None
    pub, _, _ = recover_transcribed(m % N, r % N, s % N, even, cap)
    return STATUS[0], output_of(address_of(pub))


# ---- the closed first-candidate rule --------------------------------------------------------------------------------------------------
def recover_closed(m, r, s, even):
    """the device's rule on reduced m, r, s: Q = r^-1 (s R - m G) for r, s != 0 and r liftable, else None (no key)"""
    if r == 0 or s == 0:
        return None
    R = lift_x(r, even)
    if R is None:
        return None
    r_inv = pow(r, -1, N)
    return ec_lincomb((-m * r_inv) % N, G, s * r_inv % N, R)


def closed(inp: bytes, r_len: int = 32):
    if len(inp) != 128:
        return STATUS[1], None
    if r_len != 32:
        return STATUS[2], None
    m, vw, r, s = parse(inp)
    even = v_check(vw)
    if even is None:
        return STATUS[7], None
    return STATUS[0], output_of(address_of(recover_closed(m % N, r % N, s % N, even)))


def batch_output(inp: bytes):
    """(status, 32 bytes) of one batch record: a malformed record reads zeros"""
    st, out = closed(inp)
    return st, out if out is not None else b"\0" * 32


# ---- designed edges ------------------------------------------------------------------------------------------------------------------
def designed_inputs(signed):
    """(name, record) pairs at the edges of the first-candidate rule, built around valid signed records (128 bytes each)"""
    rnd = random.Random(11)
    out = []
    m0, _, r0, s0 = parse(signed[0])
    v0 = signed[0][63]
    pmn = P - N

    def unliftable(lo, hi):
        while True:
            x = rnd.randrange(lo, hi)
            if lift_x(x % N, True) is None:
                return x

    for name, r in (("r=0", 0), ("r=n", N), ("r=n+1", N + 1), ("r=2^256-1", 2 ** 256 - 1),
                    ("r<p-n unliftable", unliftable(1, pmn)), ("r>=p-n unliftable", unliftable(pmn, N)),
                    ("r small unliftable", unliftable(1, 1 << 20)), ("r=n+r0", N + r0 if N + r0 < 2 ** 256 else r0)):
        out.append((name, record(m0, v0, r, s0)))
    for name, s in (("s=0", 0), ("s=n", N), ("s=n+s0", (N + s0) if N + s0 < 2 ** 256 else s0), ("s=2^256-1", 2 ** 256 - 1),
                    ("s=n-s0 (other half)", N - s0)):
        out.append((name, record(m0, v0, r0, s)))
    for name, m in (("m=0", 0), ("m=n", N), ("m=2^256-1", 2 ** 256 - 1), ("m=m0+n", m0 + N if m0 + N < 2 ** 256 else m0)):
        out.append((name, record(m, v0, r0, s0)))
    # Q = infinity: R = kG, r = x(R), m = s k  =>  s R - m G = 0
    for k in (2, 3, rnd.randrange(1, N)):
        R = ec_mul(k, G)
        if R[0] >= N:
            continue
        s = rnd.randrange(1, N)
        out.append(("Q=inf k=%d" % k, record(s * k % N, 27 + (R[1] & 1), R[0], s)))
        out.append(("Q=inf other parity k=%d" % k, record(s * k % N, 28 - (R[1] & 1), R[0], s)))
    for v in (0, 1, 27, 28):
        out.append(("v=%d" % v, record(m0, v, r0, s0)))
    return out


# ---- signatures in bulk -------------------------------------------------------------------------------------------------------------
def bulk_records(count, seed=1, keys=16, nonces=16):
    """count valid (record, address) pairs from a few fixed keys d and nonces k: kG is computed once per nonce, then each record
    needs scalar arithmetic only: s = k^-1 (m + r d) mod n, v = 27 + parity of y(kG) (nonces with x(kG) >= n are skipped)."""
    rnd = random.Random(seed)
    ds = [rnd.randrange(1, N) for _ in range(keys)]
    addrs = [address_of(ec_mul(d, G)) for d in ds]
    ks = []
    while len(ks) < nonces:
        k = rnd.randrange(1, N)
        R = ec_mul(k, G)
        if R[0] < N:
            ks.append((k, pow(k, -1, N), R[0], 27 + (R[1] & 1)))
    vw = [v.to_bytes(32, "big") for v in (27, 28)]
    recs, want = [], []
    for _ in range(count):
        j = rnd.randrange(keys)
        k, k_inv, r, v = ks[rnd.randrange(nonces)]
        m = rnd.getrandbits(256)
        s = k_inv * (m + r * ds[j]) % N
        recs.append(m.to_bytes(32, "big") + vw[v - 27] + r.to_bytes(32, "big") + s.to_bytes(32, "big"))
        want.append(addrs[j])
    return recs, want
