#!/usr/bin/env python3
"""Build tests/golden/evm_modexp_hashes_kat.json (the fixture, not this script, is what the tests read).

Sources:
  - the reference's tests/protocol_ethereum_evm_precompiles/modexp.json and modexp_eip2565.json (the EIP-198 examples and the
    nagydani vectors, moduli of 32 to 1024 bytes; Expected is the result);
  - the 18 audit inputs of the reference's tests/t_ethereum_evm_modexp.nim, parsed from the Nim source, with the output length,
    the status and, where the test asserts one, the result;
  - the 9 RIPEMD-160 vectors of the reference's tests/t_hash_ripemd160_vs_openssl.nim, including a million "a"s;
  - SHA-256 (hashlib) and RIPEMD-160 (hashlib when OpenSSL provides it, else the pure-Python model, which the 9 vectors check)
    digests of the seeded messages evm_modexp_exact.hash_message(n) for every n in evm_modexp_exact.hash_lengths().
Usage: make_evm_modexp_hashes_golden.py [reference tests directory]
"""
import hashlib
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import evm_modexp_exact as E  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/tests"


def json_vectors():
    out = []
    for fn in ("modexp.json", "modexp_eip2565.json"):
        with open(os.path.join(REF, "protocol_ethereum_evm_precompiles", fn)) as f:
            for v in json.load(f):
                out.append({"name": "%s:%s" % (fn, v["Name"]), "source": fn, "input": v["Input"], "out_len": len(v["Expected"]) // 2,
                            "status": "cttEVM_Success", "expected": v["Expected"]})
    return out


def _nim_bytes(body):
    body = re.sub(r"#[^\n]*", "", body).replace("uint8", "")
    return bytes(int(t, 0) for t in re.findall(r"0x[0-9a-fA-F]+|\b\d+\b", body))


def audit_vectors():
    with open(os.path.join(REF, "t_ethereum_evm_modexp.nim")) as f:
        src = f.read()
    out = []
    for m in re.finditer(r'test "([^"]+)":(.*?)(?=\n  test "|\Z)', src, re.S):
        name, body = m.group(1), m.group(2)
        inp = _nim_bytes(re.search(r"input = @\[(.*?)\]", body, re.S).group(1))
        out_len = int(re.search(r"newSeq\[byte\]\((0x[0-9a-fA-F]+|\d+)\)", body).group(1), 0)
        status = re.search(r"status == (cttEVM_\w+)", body).group(1)
        exp = None
        full = re.search(r"doAssert r == @\[byte ([^\]]*)\]", body)
        if full:
            exp = bytes(int(t, 0) for t in full.group(1).split(","))
        elif re.search(r"doAssert r\[0\] == 0", body):
            exp = bytes(out_len) if out_len == 1 else None
        out.append({"name": "audit:" + name, "source": "audit", "input": inp.hex(), "out_len": out_len, "status": status,
                    "expected": exp.hex() if exp is not None else None})
    return out


RIPEMD_REF = [
    (b"", "9c1185a5c5e9fc54612808977ee8f548b2258d31"),
    (b"a", "0bdc9d2d256b3ee9daae347be6f4dc835a467ffe"),
    (b"abc", "8eb208f7e05d987a9b044a8e98c6b087f15a0bfc"),
    (b"message digest", "5d0689ef49d2fae572b881b123a85ffa21595f36"),
    (b"abcdefghijklmnopqrstuvwxyz", "f71c27109c692c1b56bbdceb5b9d2865b3708dbc"),
    (b"abcdbcdecdefdefgefghfghighijhijkijkljklmklmnlmnomnopnopq", "12a053384a9c0c88e405a06c27dcf49ada62eb2b"),
    (b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789", "b0e20b6e3116640286ed3a87a5713079b21f5189"),
    (b"1234567890" * 8, "9b752e45573d4b39f4dbd3323cab82bf63326bfb"),
    (b"a" * 1000000, "52783243c1697bdbe16d37f97f68f08325dc1528"),
]


def ripemd(msg):
    try:
        return hashlib.new("ripemd160", msg).digest()
    except ValueError:
        return E.ripemd160(msg)


def hash_vectors():
    out = []
    for n in E.hash_lengths():
        msg = E.hash_message(n)
        out.append({"len": n, "sha256": hashlib.sha256(msg).hexdigest(), "ripemd160": ripemd(msg).hex()})
    return out


if __name__ == "__main__":
    for msg, want in RIPEMD_REF:
        assert E.ripemd160(msg).hex() == want
    data = {"modexp": json_vectors() + audit_vectors(),
            "ripemd160_reference": [{"message": m.hex() if len(m) < 1000 else None, "repeat_a": len(m) if len(m) >= 1000 else None,
                                     "digest": d} for m, d in RIPEMD_REF],
            "hashes": hash_vectors()}
    with open(os.path.join(HERE, "evm_modexp_hashes_kat.json"), "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")
    print("wrote %d modexp vectors, %d hash lengths" % (len(data["modexp"]), len(data["hashes"])))
