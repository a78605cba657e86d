#!/usr/bin/env python3
"""Build tests/golden/eth_ecdsa_kat.json (the fixture, not this script, is what the tests read).

Made with OpenSSL through the `cryptography` package, and with the exact model (tests/eth_ecdsa_exact.py) where OpenSSL has no
counterpart:
  - keys: 8 seeded secret keys and their public keys (OpenSSL's, checked against the model);
  - lengths: messages of every length 0..300 (the Keccak rate boundaries 135/136/137 and 271/272/273 among them), 1 KB and
    64 KB; the bytes are eth_ecdsa_exact.fixture_message(length), a SHAKE-256 expansion, so only the lengths are stored;
  - openssl_random: every message signed by OpenSSL with a random nonce over its Keccak-256 digest (s as OpenSSL returns it, low
    or high);
  - openssl_rfc6979_sha256: OpenSSL's deterministic (RFC 6979) signatures over SHA-256 digests, which pin the model's DRBG;
  - model_rfc6979_keccak: the model's RFC 6979 signatures with Keccak-256 and HMAC over 200-byte blocks (the reference's nonces,
    which no other library makes), each accepted by OpenSSL's verify.
`cryptography` is needed only here.
"""
import hashlib
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import eth_ecdsa_exact as X  # noqa: E402

LENGTHS = list(range(0, 301)) + [1024, 65536]


def main():
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec
    from cryptography.hazmat.primitives.asymmetric.utils import Prehashed, decode_dss_signature, encode_dss_signature

    rnd = random.Random(4242)
    ds = [rnd.randrange(1, X.N) for _ in range(8)]
    sks = [ec.derive_private_key(d, ec.SECP256K1()) for d in ds]
    keys = []
    for d, sk in zip(ds, sks):
        pn = sk.public_key().public_numbers()
        assert X.derive_pubkey(d.to_bytes(32, "big"))[1] == X.pub_bytes((pn.x, pn.y))
        keys.append({"secret_key": "%064x" % d, "pubkey": "%064x%064x" % (pn.x, pn.y)})
    msgs = [X.fixture_message(n) for n in LENGTHS]
    prehashed = ec.ECDSA(Prehashed(hashes.SHA256()))

    openssl_random, model_keccak = [], []
    for i, m in enumerate(msgs):
        j = i % len(ds)
        digest = X.keccak256(m)
        r, s = decode_dss_signature(sks[j].sign(digest, prehashed))
        sig = r.to_bytes(32, "big") + s.to_bytes(32, "big")
        assert X.verify(bytes.fromhex(keys[j]["pubkey"]), m, sig) == X.SUCCESS
        openssl_random.append({"key": j, "msg": i, "digest": digest.hex(), "sig": sig.hex(), "high_s": s > X.N // 2})
        st, sig = X.sign(ds[j].to_bytes(32, "big"), m, X.NONCE_RFC6979)
        assert st == X.SUCCESS
        r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
        sks[j].public_key().verify(encode_dss_signature(r, s), digest, prehashed)   # raises when invalid
        model_keccak.append({"key": j, "msg": i, "sig": sig.hex()})

    openssl_det = []
    det = ec.ECDSA(Prehashed(hashes.SHA256()), deterministic_signing=True)
    for i in range(64):
        d = ds[i % len(ds)] if i % 2 else rnd.randrange(1, X.N)
        digest = hashlib.sha256(rnd.randbytes(i)).digest()
        r, s = decode_dss_signature(ec.derive_private_key(d, ec.SECP256K1()).sign(digest, det))
        openssl_det.append({"secret_key": "%064x" % d, "digest": digest.hex(), "r": "%064x" % r, "s": "%064x" % s})

    data = {"keys": keys, "lengths": LENGTHS, "openssl_random": openssl_random, "openssl_rfc6979_sha256": openssl_det,
            "model_rfc6979_keccak": model_keccak}
    with open(os.path.join(HERE, "eth_ecdsa_kat.json"), "w") as f:   # one entry per line
        rows = lambda v: "[\n%s\n]" % ",\n".join(json.dumps(e) for e in v)   # noqa: E731
        f.write("{\n" + ",\n".join('"%s": %s' % (k, json.dumps(v) if k == "lengths" else rows(v)) for k, v in data.items()) + "\n}\n")
    print("wrote %d messages, %d + %d + %d signatures" % (len(msgs), len(openssl_random), len(openssl_det), len(model_keccak)))


if __name__ == "__main__":
    main()
