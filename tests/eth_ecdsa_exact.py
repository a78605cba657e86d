"""Exact model of Ethereum ECDSA over secp256k1 as this library computes it (constantine_b200/csrc/eth_ecdsa.cu), written from the
reference's Nim source (constantine/signatures/ecdsa.nim, constantine/ethereum_ecdsa_signatures.nim, constantine/mac/mac_hmac.nim)
and the definitions (SEC 1, RFC 6979, Keccak-256). The curve and Keccak code is evm_ecrecover_exact's.

Two layers:
  - the reference transcribed: hmac(), nonce_rfc6979(), sign_impl(), verify_impl() and recover_impl() with the hash and its
    block size as parameters and the reference's conventions (Fr inv(0) = 0, the affine (0, 0) is infinity); its unbounded loops
    run under explicit caps;
  - the byte API of the library's entries on top of it: 32-byte secret keys, 64-byte public keys x || y and signatures r || s,
    big-endian, with a status per item (STATUS), r = 0 and s = 0 rejected up front in verify (the one deliberate deviation), and
    recovery by ECRECOVER's first-candidate rule (evm_ecrecover_exact.recover_closed), which gives recover_impl's result whenever
    that returns.
Plus the fixed-base table and the complete addition the signing kernel uses, to check them against the plain group law.
"""
import hashlib

import evm_ecrecover_exact as E
from evm_ecrecover_exact import B, G, N, P, ec_add, ec_mul, keccak256, lift_x, on_curve

STATUS = ("cttEthEcdsa_Success", "cttEthEcdsa_VerificationFailure", "cttEthEcdsa_SecretKeyOutOfRange",
          "cttEthEcdsa_SignatureOutOfRange", "cttEthEcdsa_PublicKeyCoordinateOutOfRange", "cttEthEcdsa_PublicKeyNotOnCurve",
          "cttEthEcdsa_NonceFailure")
(SUCCESS, VERIFICATION_FAILURE, SECRET_KEY_OUT_OF_RANGE, SIGNATURE_OUT_OF_RANGE, PUBKEY_COORDINATE_OUT_OF_RANGE,
 PUBKEY_NOT_ON_CURVE, NONCE_FAILURE) = STATUS
NONCE_RANDOM, NONCE_RFC6979 = 0, 1       # the reference's NonceSampler order: nsRandom, nsRfc6979
KECCAK_BLOCK = 200                       # h_keccak.nim internalBlockSize: the whole state, not the 136-byte rate
NONCE_ROUNDS = 8                         # the library's bound on step h of RFC 6979


def sha256(m: bytes) -> bytes:
    return hashlib.sha256(m).digest()


# ---- the reference transcribed ----------------------------------------------------------------------------------------------------
def hmac(H, block, key: bytes, msg: bytes) -> bytes:
    """mac_hmac.nim: a key longer than the block is hashed first; the key is zero-padded to `block` bytes"""
    if len(key) > block:
        key = H(key)
    key = key + b"\0" * (block - len(key))
    inner = H(bytes(b ^ 0x36 for b in key) + msg)
    return H(bytes(b ^ 0x5C for b in key) + inner)


def nonce_rfc6979(z, d, H=keccak256, block=KECCAK_BLOCK, rounds=None):
    """nonceRfc6979(msgHash = z, privateKey = d) (ecdsa.nim:104-166): the nonce, or None when step h has run `rounds` times
    without a candidate in [1, n - 1] (the reference loops for ever; rounds=None does too)"""
    x, h = d.to_bytes(32, "big"), z.to_bytes(32, "big")
    v, k = b"\x01" * 32, b"\0" * 32
    k = hmac(H, block, k, v + b"\0" + x + h)
    v = hmac(H, block, k, v)
    k = hmac(H, block, k, v + b"\x01" + x + h)
    v = hmac(H, block, k, v)
    tried = 0
    while rounds is None or tried < rounds:
        tried += 1
        v = hmac(H, block, k, v)
        cand = int.from_bytes(v, "big")
        if cand != 0 and cand < N:
            return cand
        k = hmac(H, block, k, v + b"\0")
        v = hmac(H, block, k, v)
    return None


def inv_n(a):
    return pow(a, -1, N) if a % N else 0          # Fr inv: 0^-1 = 0


def sign_impl(d, z, nonces, cap=4):
    """signImpl (ecdsa.nim:175-226) with the nonces drawn from the iterator `nonces`: (r, s), low-s normalized, or None after
    `cap` nonces that gave r = 0 or s = 0 (the reference retries for ever)"""
    for _ in range(cap):
        k = next(nonces)
        R = ec_mul(k, G)
        r = (R[0] if R is not None else 0) % N
        if r == 0:
            continue
        s = inv_n(k) * (z + r * d) % N
        if s > N - s:
            s = N - s
        if s == 0:
            continue
        return r, s
    return None


def verify_impl(pub, r, s, z):
    """verifyImpl (ecdsa.nim:258-291): pub affine (None or (0, 0) for infinity), r and s elements of Fr (0 allowed)"""
    return E.verify_impl(pub if pub is not None else (0, 0), r, s, z)


def recover_impl(z, r, s, even, cap=64):
    """recoverPubkeyImpl_vartime (ecdsa.nim:311-382): the recovered key, None for the neutral element"""
    return E.recover_transcribed(z, r, s, even, cap)[0]


def fixture_message(n: int) -> bytes:
    """the n-byte message of tests/golden/eth_ecdsa_kat.json, which stores only the lengths"""
    return hashlib.shake_256(b"eth_ecdsa_kat %d" % n).digest(n)


def digest_scalar(digest: bytes) -> int:
    """fromDigest(truncateInput = true) of a 32-byte digest: the big-endian integer mod n (no shift: n has 256 bits)"""
    return int.from_bytes(digest, "big") % N


# ---- the byte API ----------------------------------------------------------------------------------------------------------------
def pub_bytes(pt) -> bytes:
    x, y = pt if pt is not None else (0, 0)
    return x.to_bytes(32, "big") + y.to_bytes(32, "big")


ZERO_PUB = b"\0" * 64
ZERO_SIG = b"\0" * 64


def _secret(sk: bytes):
    d = int.from_bytes(sk, "big")
    return d if 0 < d < N else None


def _signature(sig: bytes):
    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
    return (r, s) if 0 < r < N and 0 < s < N else None


def _pubkey(pub: bytes):
    """(status, point)"""
    x, y = int.from_bytes(pub[:32], "big"), int.from_bytes(pub[32:], "big")
    if x >= P or y >= P:
        return PUBKEY_COORDINATE_OUT_OF_RANGE, None
    if (y * y - x ** 3 - B) % P:
        return PUBKEY_NOT_ON_CURVE, None       # (0, 0) included: 7 is not a square
    return SUCCESS, (x, y)


def derive_pubkey(sk: bytes):
    d = _secret(sk)
    if d is None:
        return SECRET_KEY_OUT_OF_RANGE, ZERO_PUB
    return SUCCESS, pub_bytes(ec_mul(d, G))


def sign_digest(sk: bytes, digest: bytes, nonce=NONCE_RFC6979):
    """nonce: NONCE_RFC6979 or an explicit k (what the random sampler drew). -> (status, 64-byte signature)"""
    d = _secret(sk)
    if d is None:
        return SECRET_KEY_OUT_OF_RANGE, ZERO_SIG
    z = digest_scalar(digest)
    k = nonce_rfc6979(z, d, rounds=NONCE_ROUNDS) if nonce == NONCE_RFC6979 else nonce
    if k is None:
        return NONCE_FAILURE, ZERO_SIG
    rs = sign_impl(d, z, iter([k]), cap=1)
    if rs is None:
        return NONCE_FAILURE, ZERO_SIG
    return SUCCESS, rs[0].to_bytes(32, "big") + rs[1].to_bytes(32, "big")


def sign(sk: bytes, msg: bytes, nonce=NONCE_RFC6979):
    return sign_digest(sk, keccak256(msg), nonce)


def verify_digest(pub: bytes, digest: bytes, sig: bytes):
    st, q = _pubkey(pub)
    if st != SUCCESS:
        return st
    rs = _signature(sig)
    if rs is None:
        return SIGNATURE_OUT_OF_RANGE
    return SUCCESS if verify_impl(q, rs[0], rs[1], digest_scalar(digest)) else VERIFICATION_FAILURE


def verify(pub: bytes, msg: bytes, sig: bytes):
    return verify_digest(pub, keccak256(msg), sig)


def recover_from_digest(digest: bytes, sig: bytes, even_y: bool):
    rs = _signature(sig)
    if rs is None:
        return SIGNATURE_OUT_OF_RANGE, ZERO_PUB
    q = E.recover_closed(digest_scalar(digest), rs[0], rs[1], bool(even_y))   # the first candidate only (DESIGN §4s)
    if q is None:
        return VERIFICATION_FAILURE, ZERO_PUB
    return SUCCESS, pub_bytes(q)


def recover(msg: bytes, sig: bytes, even_y: bool):
    return recover_from_digest(keccak256(msg), sig, even_y)


def reference_verify_bytes(pub: bytes, msg: bytes, sig: bytes) -> bool:
    """what the reference's verify returns when handed these bytes as they are (r and s taken into Fr with no range check, the
    key as given): the behaviour the byte API deviates from at r = 0 and s = 0"""
    x, y = int.from_bytes(pub[:32], "big"), int.from_bytes(pub[32:], "big")
    r, s = int.from_bytes(sig[:32], "big") % N, int.from_bytes(sig[32:], "big") % N
    return verify_impl((x, y), r, s, digest_scalar(keccak256(msg)))


# ---- the signing kernel's group law and table ----------------------------------------------------------------------------------------
B3 = 3 * B


def rcb_add(p, q):
    """Renes-Costello-Batina 2016, Algorithm 7 (complete addition, a = 0) on projective (X : Y : Z); (0 : 1 : 0) is infinity"""
    X1, Y1, Z1 = p
    X2, Y2, Z2 = q
    t0 = X1 * X2 % P; t1 = Y1 * Y2 % P; t2 = Z1 * Z2 % P
    t3 = (X1 + Y1) * (X2 + Y2) % P; t4 = (t0 + t1) % P; t3 = (t3 - t4) % P
    t4 = (Y1 + Z1) * (Y2 + Z2) % P; X3 = (t1 + t2) % P; t4 = (t4 - X3) % P
    X3 = (X1 + Z1) * (X2 + Z2) % P; Y3 = (t0 + t2) % P; Y3 = (X3 - Y3) % P
    X3 = (t0 + t0) % P; t0 = (X3 + t0) % P; t2 = B3 * t2 % P
    Z3 = (t1 + t2) % P; t1 = (t1 - t2) % P; Y3 = B3 * Y3 % P
    X3 = t4 * Y3 % P; t2 = t3 * t1 % P; X3 = (t2 - X3) % P
    Y3 = Y3 * t0 % P; t1 = t1 * Z3 % P; Y3 = (t1 + Y3) % P
    t0 = t0 * t3 % P; Z3 = Z3 * t4 % P; Z3 = (Z3 + t0) % P
    return X3, Y3, Z3


def proj_to_affine(p):
    if p[2] == 0:
        return None
    zi = pow(p[2], -1, P)
    return p[0] * zi % P, p[1] * zi % P


WINDOWS, ENTRIES = 64, 15                # [j 16^i]G for i < 64, j = 1..15


def fixed_base_table():
    """rows[i][j - 1] = [j 16^i]G, affine"""
    rows, base = [], G
    for _ in range(WINDOWS):
        row, acc = [], None
        for _ in range(ENTRIES):
            acc = ec_add(acc, base)
            row.append(acc)
        rows.append(row)
        base = ec_add(row[-1], base)      # 16 * base
    return rows


def fixed_base_mul(k, rows):
    """the kernel's [k]G: one complete addition per 4-bit window, the selected entry (0 : 1 : 0) for a zero digit"""
    acc = (0, 1, 0)
    for i in range(WINDOWS):
        d = (k >> (4 * i)) & 15
        sel = (rows[i][d - 1][0], rows[i][d - 1][1], 1) if d else (0, 1, 0)
        acc = rcb_add(acc, sel)
    return proj_to_affine(acc)


__all__ = ["STATUS", "G", "N", "P", "lift_x", "on_curve", "keccak256"]
