"""CPU: a SASS audit of the constant-time subroutines of the signing and key-derivation kernels (secp256k1_ct.cuh, bls_ct.cuh,
eip2333.cuh; DESIGN §4v, §4w, §4x).

Those files promise that no branch and no memory address depends on secret data. The arithmetic they run is shared with the
variable-time code (field.cuh's Fp, the secp256k1 products), and whether a select stays a SEL or becomes a jump is the compiler's
choice, so the promise is checked on the machine code the build produced: `cuobjdump -xelf all` of libctt_b200_msm.so, `nvdisasm -c`
of the three cubins that hold the kernels, one body per `.type` (a `__noinline__` subroutine appears once per calling kernel, as
`$<kernel>$<callee>`), names demangled by `cu++filt`.

For every production kernel below the audited subroutines must be present, call nothing outside the audited set, use no indirect
branch, branch exactly as the tables below say (each count names its loop or its public condition), and predicate no memory
instruction except where a public length decides it. The counts are exact on purpose: the toolkit is pinned (CUDA 12.9, sm_90a),
and a compiler or source change that moves them sends someone back to read the SASS before the tables are updated.
"""
import functools
import os
import re
import shutil
import subprocess
import tempfile
from collections import namedtuple

import pytest

from helpers import ROOT

# ---- the tools of the toolkit that built the library -------------------------------------------------------------------------------


def _cuda_bin():
    """the directory of the nvcc the Makefile runs (`nvcc` on PATH, else CUDA_HOME or /usr/local/cuda)"""
    nvcc = shutil.which("nvcc")
    if nvcc:
        return os.path.dirname(os.path.realpath(nvcc))
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.path.isfile(os.path.join(home, "bin", "nvcc")):
            return os.path.join(home, "bin")
    return None


def _tool(name):
    d = _cuda_bin()
    if d is None:
        pytest.skip("no CUDA toolkit (nvcc) found: the SASS audit needs cuobjdump, nvdisasm and cu++filt")
    path = os.path.join(d, name)
    if not os.access(path, os.X_OK):
        pytest.skip("%s is absent next to nvcc in %s" % (name, d))
    return path


# ---- the listing -------------------------------------------------------------------------------------------------------------------
Inst = namedtuple("Inst", "addr pred op text")      # pred: the guard ("@P0", "@!P1", ...) or ""
Body = namedtuple("Body", "insts labels")           # labels: .L_x_N -> address of the next instruction

_TYPE = re.compile(r"^\s*\.type\s+(\S+),@function")
_INST = re.compile(r"^\s*/\*([0-9a-f]+)\*/\s+(.*?)\s*;")
_LABEL = re.compile(r"^(\.L_x_\d+):")
_TARGET = re.compile(r"`\((\.L_x_\d+)\)")
_CALLEE = re.compile(r"`\((\$[^)]+)\)")


def _split(listing):
    """mangled symbol -> Body, one per `.type` of the listing"""
    bodies, name, insts, labels, pending = {}, None, [], {}, []

    def flush():
        if name is not None:
            end = insts[-1].addr + 16 if insts else 0
            for lab in pending:
                labels[lab] = end
            bodies[name] = Body(list(insts), dict(labels))

    for line in listing.splitlines():
        m = _TYPE.match(line)
        if m or line.startswith("//----"):
            flush()
            name, insts, labels, pending = (m.group(1) if m else None), [], {}, []
            continue
        m = _LABEL.match(line)
        if m:
            pending.append(m.group(1))
            continue
        m = _INST.match(line)
        if m and name is not None:
            addr, text = int(m.group(1), 16), m.group(2)
            for lab in pending:
                labels[lab] = addr
            pending = []
            pred = ""
            if text.startswith("@"):
                pred, text = text.split(None, 1)
            insts.append(Inst(addr, pred, text.split()[0], text))
    flush()
    return bodies


def _demangle(names):
    out = subprocess.run([_tool("cu++filt")], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    return dict(zip(names, out.splitlines()))


def _base(demangled):
    """`b200::blsct::ct_fp_inv(b200::Fp<...>)` -> `b200::blsct::ct_fp_inv`, the qualified name without the parameters"""
    depth = 0
    for i, ch in enumerate(demangled):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0 and not demangled.startswith("(anonymous", i):
            return demangled[:i]
    return demangled


def _short(qualified):
    """the last component of a qualified name (template arguments kept apart)"""
    depth, start = 0, 0
    for i, ch in enumerate(qualified):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif depth == 0 and qualified.startswith("::", i):
            start = i + 2
    return qualified[start:]


MUL_CALL = "b200::Fp<b200::Bls12381Fp>::mul_call"


def _audited_name(qualified):
    """the audit's name of a subroutine, or None when it is outside the audited set"""
    if qualified == MUL_CALL:
        return "mul_call"
    s = _short(qualified)
    return s if s.startswith("ct_") else None


Sub = namedtuple("Sub", "name qualified body calls")   # calls: audited names of the CALL targets, or qualified names outside the set

UNITS = ("eth_ecdsa", "eth_bls_sign", "eth_bls_keygen")


@functools.lru_cache(maxsize=None)
def _subroutines():
    """(unit, kernel) -> {name: Sub} for every subroutine of every kernel of the three translation units"""
    from constantine_b200 import _lib
    lib = _lib.LIB_PATH
    assert os.path.isfile(lib), "libctt_b200_msm.so is not built (run __graft_entry__.build())"
    cuobjdump, nvdisasm = _tool("cuobjdump"), _tool("nvdisasm")
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([cuobjdump, "-xelf", "all", lib], cwd=tmp, check=True, capture_output=True)
        listings = {}
        for unit in UNITS:
            cubins = [f for f in os.listdir(tmp) if f.startswith(unit + ".") and f.endswith(".cubin")]
            assert len(cubins) == 1, (unit, sorted(os.listdir(tmp)))
            listings[unit] = subprocess.run([nvdisasm, "-c", os.path.join(tmp, cubins[0])], check=True, capture_output=True,
                                            text=True).stdout
    result = {}
    for unit, listing in listings.items():
        bodies = _split(listing)
        names = set()
        for sym in bodies:
            names.update(p for p in sym.split("$") if p)
        for body in bodies.values():
            for ins in body.insts:
                names.update(c.lstrip("$").split("$")[-1] for c in _CALLEE.findall(ins.text))
        dm = {k: _base(v) for k, v in _demangle(sorted(names)).items()}
        for sym, body in bodies.items():
            if not sym.startswith("$"):
                continue
            kernel, callee = sym[1:].split("$")
            calls = []
            for ins in body.insts:
                if ins.op.startswith("CALL"):
                    for c in _CALLEE.findall(ins.text):
                        q = dm[c[1:].split("$")[-1]]
                        calls.append(_audited_name(q) or q)
            q = dm[callee]
            key = (unit, _short(dm[kernel]))
            result.setdefault(key, {})[_audited_name(q) or q] = Sub(_audited_name(q), q, body, tuple(calls))
    return result


# ---- what a body does ----------------------------------------------------------------------------------------------------------------
Branches = namedtuple("Branches", "backward forward conditional indirect")


def branches(body):
    """BRA classified by its resolved target: backward, forward (the self-branch that parks a lane after the return is neither),
    conditional (predicated, any direction); indirect counts BRX / JMX"""
    back = fwd = cond = ind = 0
    for ins in body.insts:
        if ins.op.startswith(("BRX", "JMX")):
            ind += 1
        if not ins.op.startswith("BRA"):
            continue
        m = _TARGET.search(ins.text)
        assert m, ins.text
        target = body.labels[m.group(1)]
        if ins.pred:
            cond += 1
        if target < ins.addr:
            back += 1
        elif target > ins.addr:
            fwd += 1
        else:
            assert not ins.pred, ins.text
    return Branches(back, fwd, cond, ind)


_MEM = re.compile(r"^(LDG|STG|LDL|STL|LDS|STS|LD|ST)(\.|$)")


def predicated_memory(body):
    return [ins for ins in body.insts if ins.pred and _MEM.match(ins.op)]


# ---- what the build must contain -----------------------------------------------------------------------------------------------------
K1_DERIVE = {"ct_fixed_base_mul", "ct_point_add", "ct_select", "ct_fp_inv"}
G1_DERIVE = {"ct_fixed_base_g1", "ct_g1_add", "ct_g1_select", "ct_fp_inv", "mul_call"}
KERNELS = {
    ("eth_ecdsa", "k_ecdsa_sign"): K1_DERIVE | {"ct_rfc6979_nonce", "ct_hmac_keccak256", "ct_fr_inv"},
    ("eth_ecdsa", "k_ecdsa_derive"): K1_DERIVE,
    ("eth_bls_sign", "k_bls_sign"): {"ct_mul_g2", "ct_g2_dbl", "ct_g2_add", "ct_g2_select", "ct_fp2_inv", "ct_fp_inv", "mul_call"},
    ("eth_bls_sign", "k_bls_derive"): G1_DERIVE,
    ("eth_bls_keygen", "k_bls_derive"): G1_DERIVE,
    ("eth_bls_keygen", "k_eip2333_child"): {"ct_derive_child", "ct_reduce_mod_r"},
    ("eth_bls_keygen", "k_eip2333_master"): {"ct_derive_master", "ct_reduce_mod_r"},
}

# (backward, forward) BRA per function, the self-branch after the return not counted. No entry may branch on secret data.
BRANCHES = {
    # straight-line: no branch at all
    "ct_point_add": (0, 0), "ct_g1_add": (0, 0), "ct_g2_add": (0, 0), "ct_g2_dbl": (0, 0), "ct_fp2_inv": (0, 0),
    "ct_reduce_mod_r": (0, 0), "mul_call": (0, 0),
    # loops with fixed trip counts: one backward branch per loop, nothing forward
    "ct_fp_inv": (3, 0),              # the table a^0..a^15, the 4-bit windows of the exponent, the four squarings of a window
    "ct_fr_inv": (3, 0),              # the same three loops
    "ct_select": (1, 0),              # the 15 entries of a row
    "ct_g1_select": (1, 0),           # the 15 entries of a row
    "ct_g2_select": (1, 0),           # the 15 entries of the caller's table
    "ct_fixed_base_mul": (1, 0),      # the 64 windows
    "ct_fixed_base_g1": (1, 0),       # the 64 windows
    "ct_mul_g2": (2, 0),              # the 63 windows, the four doublings of a window
    # the DRBG and the key derivations: forward branches on public data only (DESIGN §4v, §4x)
    "ct_hmac_keccak256": (8, 6),      # back: the two pad loops, the digest and tag copies, and per hash its block and round loops;
                                      # forward: keccak256_bytes' full-block test and the last block's `at < len`, on the public
                                      # message length, and the key's `i < 32` on the loop counter
    "ct_rfc6979_nonce": (13, 4),      # back: the DRBG's byte-copy loops at each call site, step h's candidate loop, the wipes;
                                      # forward: the reference's candidate test (step h.3) leaving the loop, and its bound
    "ct_derive_child": (27, 4),       # back: the round loops of the SHA-256 compressions and the chain loops; forward: the
                                      # chain's i == 1 case (2), the parity of the digest count and the SK = 0 retry
    "ct_derive_master": (13, 4),      # back: the round and block loops of sha256_from and the HMACs, the SK = 0 retry's jump back;
                                      # forward: sha256_from's full-block and last-block tests on the public length (3) and the
                                      # SK = 0 retry
}
# memory instructions under a predicate: only where the public message length decides which bytes are read
PREDICATED_MEMORY = {"ct_hmac_keccak256": 271, "ct_derive_master": 64}


@pytest.fixture(scope="module")
def subs():
    return _subroutines()


def _kernel_ids():
    return ["%s:%s" % k for k in KERNELS]


def test_tables_cover_every_audited_function():
    named = set().union(*KERNELS.values())
    assert named == set(BRANCHES), sorted(named ^ set(BRANCHES))
    assert set(PREDICATED_MEMORY) <= named


@pytest.mark.parametrize("key", list(KERNELS), ids=_kernel_ids())
def test_audited_subroutines_are_present(subs, key):
    """Each kernel calls its constant-time functions as separate subroutines: a dropped __noinline__ or a renamed function must
    fail here, not leave the audit with nothing to read."""
    assert key in subs, "kernel %s not found in %s" % (key[1], key[0])
    audited = {name for name, s in subs[key].items() if s.name is not None}
    assert audited == KERNELS[key], "missing %s, unexpected %s" % (sorted(KERNELS[key] - audited), sorted(audited - KERNELS[key]))


@pytest.mark.parametrize("key", list(KERNELS), ids=_kernel_ids())
def test_audited_calls_stay_inside_the_set(subs, key):
    bad = {(name, c) for name in KERNELS[key] if name in subs[key] for c in subs[key][name].calls if c not in KERNELS[key]}
    assert not bad, sorted(bad)


@pytest.mark.parametrize("key", list(KERNELS), ids=_kernel_ids())
def test_branches_match_the_table(subs, key):
    """No indirect branch; straight-line functions no branch at all; loops only their backward branches; the DRBG and the key
    derivations exactly their documented forward branches."""
    bad = []
    for name in sorted(KERNELS[key]):
        if name not in subs[key]:
            continue
        b = branches(subs[key][name].body)
        want = BRANCHES[name]
        if b.indirect or (b.backward, b.forward) != want or (want == (0, 0) and b.conditional):
            bad.append("%s: %d backward, %d forward, %d conditional, %d indirect; want %d backward, %d forward" % (
                name, b.backward, b.forward, b.conditional, b.indirect, want[0], want[1]))
    assert not bad, "; ".join(bad)


@pytest.mark.parametrize("key", list(KERNELS), ids=_kernel_ids())
def test_no_predicated_memory_access(subs, key):
    bad = []
    for name in sorted(KERNELS[key]):
        if name not in subs[key]:
            continue
        got = predicated_memory(subs[key][name].body)
        if len(got) != PREDICATED_MEMORY.get(name, 0):
            bad.append("%s: %d predicated memory instructions, want %d (first: %s)" % (
                name, len(got), PREDICATED_MEMORY.get(name, 0), got[0].pred + " " + got[0].text if got else "-"))
    assert not bad, "; ".join(bad)


# ---- the parser on a listing whose answer is known (no toolkit needed) --------------------------------------------------------------
_SYNTHETIC = """
//--------------------- .text.kern --------------------------
        .type           kern,@function
        /*0000*/                   CALL.REL.NOINC `($kern$_ZN4b2001ct_fooEv) ;
        /*0010*/                   EXIT ;
        .type           $kern$_ZN4b2001ct_fooEv,@function
$kern$_ZN4b2001ct_fooEv:
.L_x_1:
        /*0020*/                   IMAD R2, R3, R4, RZ ;
        /*0030*/               @P0 BRA `(.L_x_2) ;
        /*0040*/               @P1 LDG.E R5, desc[UR4][R6.64] ;
        /*0050*/              @!P2 BRA `(.L_x_1) ;
.L_x_2:
        /*0060*/                   RET.REL.NODEC R20 `(kern) ;
.L_x_3:
        /*0070*/                   BRA `(.L_x_3);
"""


def test_parser_classifies_a_known_listing():
    bodies = _split(_SYNTHETIC)
    assert set(bodies) == {"kern", "$kern$_ZN4b2001ct_fooEv"}
    body = bodies["$kern$_ZN4b2001ct_fooEv"]
    assert body.labels == {".L_x_1": 0x20, ".L_x_2": 0x60, ".L_x_3": 0x70}
    assert branches(body) == Branches(backward=1, forward=1, conditional=2, indirect=0)
    assert [i.addr for i in predicated_memory(body)] == [0x40]
    assert _audited_name(_base("b200::k1::ct_foo()")) == "ct_foo"
    assert _audited_name(_base(MUL_CALL + "(b200::Fp<b200::Bls12381Fp>, b200::Fp<b200::Bls12381Fp>)")) == "mul_call"
    assert _audited_name(_base("b200::Fp<b200::Bn254SnarksFp>::mul_call(b200::Fp<b200::Bn254SnarksFp>)")) is None
    assert _audited_name(_base("b200::fe_inv_safegcd<b200::Secp256k1Fr>(unsigned int *, const unsigned int *)")) is None


if __name__ == "__main__":
    for (unit, kernel), subs in sorted(_subroutines().items()):
        for name, s in sorted(subs.items()):
            if s.name is None:
                continue
            b = branches(s.body)
            print("%-15s %-18s %-18s n=%6d back=%3d fwd=%3d cond=%3d ind=%d predmem=%d calls=%s" % (
                unit, kernel, name, len(s.body.insts), b.backward, b.forward, b.conditional, b.indirect,
                len(predicated_memory(s.body)), sorted(set(s.calls))))
