"""Exact model of EIP-2333 BLS12-381 key derivation and EIP-2334 paths over hashlib and hmac: the spec's HKDF (RFC 5869),
HKDF_mod_r, IKM_to_lamport_SK, parent_SK_to_lamport_PK, derive_child_SK and derive_master_SK, as the reference
(constantine/ethereum_eip2333_bls12381_key_derivation.nim) computes them. A child costs about 3 ms here."""
import hashlib
import hmac

R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
SALT = b"BLS-SIG-KEYGEN-SALT-"
L = 48   # ceil(1.5 ceil(log2 r) / 8)


def sha256(m):
    return hashlib.sha256(m).digest()


def hkdf_extract(salt, ikm):
    return hmac.new(salt, ikm, hashlib.sha256).digest()


def hkdf_expand(prk, info, length):
    t, okm, i = b"", b"", 1
    while len(okm) < length:
        t = hmac.new(prk, t + info + bytes([i]), hashlib.sha256).digest()
        okm += t
        i += 1
    return okm[:length]


def os2ip_mod_r(okm):
    """the device's reduction of HKDF_mod_r, exposed by the ctt_b200_test_field_op hook (field 13, op 13)"""
    return int.from_bytes(okm, "big") % R


def hkdf_mod_r(ikm, key_info=b""):
    salt, sk = SALT, 0
    while sk == 0:
        salt = sha256(salt)
        prk = hkdf_extract(salt, ikm + b"\0")
        sk = os2ip_mod_r(hkdf_expand(prk, key_info + L.to_bytes(2, "big"), L))
    return sk


def ikm_to_lamport_sk(ikm, salt):
    okm = hkdf_expand(hkdf_extract(salt, ikm), b"", 255 * 32)
    return [okm[32 * i:32 * i + 32] for i in range(255)]


def parent_sk_to_lamport_pk(parent, index):
    salt = index.to_bytes(4, "big")
    ikm = parent.to_bytes(32, "big")
    lamport_0 = ikm_to_lamport_sk(ikm, salt)
    lamport_1 = ikm_to_lamport_sk(bytes(b ^ 0xFF for b in ikm), salt)
    return sha256(b"".join(sha256(c) for c in lamport_0 + lamport_1))


def derive_child_sk(parent, index):
    return hkdf_mod_r(parent_sk_to_lamport_pk(parent, index))


def derive_master_sk(seed):
    """None for a seed shorter than 32 bytes (the reference returns false)"""
    return hkdf_mod_r(bytes(seed)) if len(seed) >= 32 else None


def derive_path(seed, indices):
    sk = derive_master_sk(seed)
    if sk is None:
        return None
    for i in indices:
        sk = derive_child_sk(sk, i)
    return sk


def path_counts(seed_of, paths):
    """(masters, children) that a path call derives when it derives every distinct prefix once"""
    masters = len(set(seed_of))
    prefixes = {(s,) + tuple(p[:k]) for s, p in zip(seed_of, paths) for k in range(1, len(p) + 1)}
    return masters, len(prefixes)
