#!/usr/bin/env python3
"""Build tests/golden/evm_ecrecover_kat.json (the fixture, not this script, is what the tests read).

Two sources:
  - the reference's tests/protocol_ethereum_evm_precompiles/ecRecover.json (5 vectors). Their "Expected" field is geth's output
    (empty for a failure); the fixture keeps it as geth_expected and stores this library's status and output beside it;
  - 320 digests signed by OpenSSL through the `cryptography` package with 8 fixed secret keys (ECDSA over a prehashed 32-byte
    digest, random nonces, s as OpenSSL returns it, low or high). Each entry stores the secret key, the public key, its address
    and v: the parity (27 / 28) whose recovery yields that key. The other parity must yield a different key; that is asserted here.
`cryptography` is needed only here. Usage: make_evm_ecrecover_golden.py [reference tests directory]
"""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import evm_ecrecover_exact as E  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/tests"


def reference_vectors():
    with open(os.path.join(REF, "protocol_ethereum_evm_precompiles", "ecRecover.json")) as f:
        vs = json.load(f)
    out = []
    for v in vs:
        inp = bytes.fromhex(v["Input"])
        st, o = E.transcribed(inp, cap=4)
        out.append({"name": v["Name"], "source": "reference", "input": inp.hex(), "status": st,
                    "output": o.hex() if o is not None else "", "geth_expected": v["Expected"]})
    return out


def openssl_vectors(count=320, keys=8, seed=2026):
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec
    from cryptography.hazmat.primitives.asymmetric.utils import Prehashed, decode_dss_signature

    rnd = random.Random(seed)
    ds = [rnd.randrange(1, E.N) for _ in range(keys)]
    sks = [ec.derive_private_key(d, ec.SECP256K1()) for d in ds]
    out = []
    for i in range(count):
        j = i % keys
        if i == 0:
            digest = bytes(32)
        elif i == 1:
            digest = b"\xff" * 32                       # m >= n
        else:
            digest = rnd.randbytes(32)
        der = sks[j].sign(digest, ec.ECDSA(Prehashed(hashes.SHA256())))
        r, s = decode_dss_signature(der)
        pub = sks[j].public_key().public_numbers()
        pub = (pub.x, pub.y)
        assert pub == E.ec_mul(ds[j], E.G)
        m = int.from_bytes(digest, "big")
        got = {v: E.recover_closed(m % E.N, r, s, v == 27) for v in (27, 28)}
        vs = [v for v in (27, 28) if got[v] == pub]
        assert len(vs) == 1 and got[27] != got[28], i
        inp = E.record(m, vs[0], r, s)
        st, o = E.closed(inp)
        assert st == "cttEVM_Success" and o[12:] == E.address_of(pub)
        out.append({"name": "openssl-%d" % i, "source": "openssl", "input": inp.hex(), "status": st, "output": o.hex(),
                    "secret_key": "%064x" % ds[j], "pubkey": "%064x%064x" % pub, "address": E.address_of(pub).hex(),
                    "v": vs[0], "high_s": s > E.N // 2})
    return out


if __name__ == "__main__":
    data = {"vectors": reference_vectors() + openssl_vectors()}
    with open(os.path.join(HERE, "evm_ecrecover_kat.json"), "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")
    print("wrote %d vectors" % len(data["vectors"]))
