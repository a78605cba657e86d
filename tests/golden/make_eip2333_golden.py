#!/usr/bin/env python3
"""Write tests/golden/eip2333_kat.json: the EIP-2333 key-derivation vectors and the HKDF-SHA-256 cases the suite checks.

  python tests/golden/make_eip2333_golden.py <constantine checkout>

Sources (inside the checkout), copied verbatim with nothing computed:
  tests/t_ethereum_eip2333_bls12381_key_derivation.nim   4 vectors: seed, master key, child index, child key (keys in decimal)
  tests/t_kdf_hkdf.nim                                    the 3 SHA-256 cases of RFC 5869: IKM, salt, info, L, PRK, OKM
"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def eip2333_vectors(text):
    out = []
    for body in re.split(r"\nproc test\d+ =\n", text)[1:]:
        seed = re.search(r'let seed = toBytes"(0x[0-9a-fA-F]+)"', body).group(1)
        master = re.search(r'let expectedMaster = "(\d+)"', body).group(1)
        index = re.search(r"let child_index = (\d+)'u32", body).group(1)
        child = re.search(r'let expectedChild = "(\d+)"', body).group(1)
        out.append({"seed": seed, "master_sk": master, "child_index": int(index), "child_sk": child})
    assert len(out) == 4, len(out)
    return out


def hkdf_cases(text):
    out = []
    for m in re.finditer(r"test (\d+): #[^\n]*\n  type HashType = sha256\n  const\n(.*?)(?=\ntest |\Z)", text, re.S):
        consts = {}
        for name, val in re.findall(r"\b(IKM|salt|info|L|PRK|OKM)\s*=\s*((?:\"[^\"]*\"\s*&?\s*)+|\d+)", m.group(2)):
            consts[name] = int(val) if val.isdigit() else "".join(re.findall(r'"([^"]*)"', val))
        out.append({"case": int(m.group(1)), **consts})
    assert len(out) == 3, len(out)
    return out


def main(checkout):
    with open(os.path.join(checkout, "tests", "t_ethereum_eip2333_bls12381_key_derivation.nim")) as f:
        eip = eip2333_vectors(f.read())
    with open(os.path.join(checkout, "tests", "t_kdf_hkdf.nim")) as f:
        hk = hkdf_cases(f.read())
    with open(os.path.join(HERE, "eip2333_kat.json"), "w") as f:
        json.dump({"eip2333": eip, "hkdf_sha256": hk}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
