"""GPU (-m gpu): the engine's stream and slot contract. ctt_b200_set_stream makes every call order itself behind the caller's stream;
the first engine slot launches on that stream itself, any other slot (taken while another thread holds the first) runs on its own
stream and is joined back to the caller's stream. ctt_b200_msm_device_digits returns with its work still queued, so the digits must
be visible to the next operation on the caller's stream, and the slot's next call must not touch the slot's scratch before that work
is done, even on another stream.

Ordering is built, never hoped for: a spin kernel (torch.cuda._sleep, sized once to ~150 ms) on the caller's stream holds back the
work queued behind it, and a helper thread that makes a blocking call on that stream behind the spin holds slot 0 until the spin
ends. Every result is compared byte for byte with a reference that does not depend on streams or slots: the closed form
[sum k_i s_i] G, a serial call's digits, or the known answers in tests/golden/."""
import ctypes
import hashlib
import json
import os
import random
import threading
import time

import numpy as np
import pytest

from helpers import CURVES, ROOT, pyref

pytestmark = pytest.mark.gpu
SPIN_MS = 150
SENTINEL = 0xA5


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
    """ctt_b200_set_stream and ctt_b200_set_concurrency are process-wide: restored to the defaults whatever the tests do."""
    import torch
    lib.ctt_b200_set_stream(None)
    lib.ctt_b200_set_concurrency(2)
    try:
        yield
    finally:
        torch.cuda.synchronize()
        lib.ctt_b200_set_stream(None)
        lib.ctt_b200_set_concurrency(2)


def set_stream(lib, s):
    lib.ctt_b200_set_stream(ctypes.c_void_p(s.cuda_stream) if s is not None else None)


@pytest.fixture(scope="module")
def spin():
    """spin(stream): queue ~SPIN_MS of busy waiting on `stream` (cycles measured once with CUDA events)."""
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
    ms = timed(cycles)
    assert 100 <= ms <= 300, ms

    def run(stream):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(cycles)
    return run


def gen_points(lib, cv, k):
    gen = b"".join(cv.fp.to_mont(c).to_bytes(cv.fp.nbytes, "little") for coord in cv.gen for c in coord)
    out = np.empty((len(k), cv.aff_bytes), dtype=np.uint8)
    assert lib.ctt_b200_scalar_mul_u64(cv.curve_id, gen, k.ctypes.data, len(k), out.ctypes.data) == 0
    return out


def random_scalars(rng, cv, n):
    s = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    s[:, 31] &= (1 << (cv.scalar_bits - 248)) - 1
    return s


def closed_form(cv, scal, k):
    """[sum s_i k_i mod r] G for points [k_i] G."""
    s_int = (int.from_bytes(scal[i].tobytes(), "little") for i in range(len(k)))
    return pyref.ec_mul_fast(sum(s * int(kk) for s, kk in zip(s_int, k)) % cv.fr.modulus, cv.gen, cv)


class Problem:
    """n closed-form terms on the device: points [k_i] G, two scalar sets A and B, and the answers of both."""

    def __init__(self, lib, curve, n, seed):
        import torch
        self.cv = cv = CURVES[curve]
        self.n = n
        rng = np.random.default_rng(seed)
        self.k = rng.integers(1, 2**63, size=n, dtype=np.uint64)
        self.pts = gen_points(lib, cv, self.k)
        self.sa, self.sb = random_scalars(rng, cv, n), random_scalars(rng, cv, n)
        self.want_a, self.want_b = closed_form(cv, self.sa, self.k), closed_form(cv, self.sb, self.k)
        self.d_p = torch.from_numpy(self.pts).cuda()
        self.d_sa, self.d_sb = torch.from_numpy(self.sa).cuda(), torch.from_numpy(self.sb).cuda()
        torch.cuda.synchronize()


_problems = {}


def problem(lib, curve, n):
    if (curve, n) not in _problems:
        _problems[(curve, n)] = Problem(lib, curve, n, n + CURVES[curve].curve_id)
    return _problems[(curve, n)]


class HoldSlot0:
    """A helper thread that holds engine slot 0 for one spin. It queues the spin on `stream` (the engine's caller stream), says that
    it is entering, then makes a blocking device MSM, which launches on slot 0 directly on that stream and returns only after the spin.
    Calls the main thread starts while the helper is inside land on another slot."""

    def __init__(self, M, spin, stream, small):
        self.M, self.spin, self.stream, self.small = M, spin, stream, small
        self.entered, self.result, self.done = threading.Event(), None, False

    def _run(self):
        p = self.small
        self.spin(self.stream)
        self.entered.set()
        self.result = self.M.msm_device_ptrs(p.cv, p.d_sa.data_ptr(), p.d_p.data_ptr(), p.n)
        self.done = True

    def __enter__(self):
        self.t = threading.Thread(target=self._run)
        self.t.start()
        assert self.entered.wait(60)
        time.sleep(0.03)           # the helper has released the GIL inside its C call and leased slot 0 microseconds later
        return self

    def assert_inside(self):
        assert self.t.is_alive() and not self.done

    def __exit__(self, *exc):
        self.t.join()
        if exc[0] is None:
            assert pyref.jac_bytes_to_affine(self.result, self.small.cv) == self.small.want_a
        return False


@pytest.fixture(scope="module")
def small(lib):
    return problem(lib, "bn254_snarks_g1", 1024)


# ---------------------------------------------------------------------------------------------------------- 1. inputs on the stream
@pytest.mark.parametrize("slot", ["direct", "other"])
@pytest.mark.parametrize("curve,n,levels", [("bls12_381_g1", 1 << 18, False), ("bls12_381_g1", 1 << 19, True),
                                            ("bls12_381_g2", 1 << 15, False), ("bls12_381_g2", 1 << 16, True)])
def test_inputs_written_on_caller_stream(M, lib, spin, small, curve, n, levels, slot):
    """The scalars of a device-pointer MSM are written on the caller's stream behind the spin, with no host synchronisation, then the
    call is made: ctt_b200_msm_device and ctt_b200_msm_device_digits + combine_window_digits must read the new scalars, on slot 0
    and on a slot that only orders itself behind the caller's stream. Sizes on both sides of the batched-affine threshold."""
    import torch
    p = problem(lib, curve, n)
    cv = p.cv
    c, W = M.plan(cv, n)
    g = M.digits_per_window(c)
    xyzz = 4 * cv.coord_bytes
    d_s = torch.empty_like(p.d_sa)
    digits = torch.empty(W * g * xyzz, dtype=torch.uint8, device="cuda")
    S = torch.cuda.Stream()
    for entry in ("msm_device", "digits"):
        d_s.copy_(p.d_sa)                 # the stale scalars: a call that does not wait computes MSM(A)
        digits.fill_(SENTINEL)
        torch.cuda.synchronize()
        set_stream(lib, S)
        try:
            holder = HoldSlot0(M, spin, S, small) if slot == "other" else None
            if holder:
                holder.__enter__()
            else:
                spin(S)
            with torch.cuda.stream(S):
                d_s.copy_(p.d_sb)
            if holder:
                holder.assert_inside()
            if entry == "msm_device":
                got = pyref.jac_bytes_to_affine(M.msm_device_ptrs(cv, d_s.data_ptr(), p.d_p.data_ptr(), n), cv)
            else:
                assert M.msm_device_digits(cv, digits.data_ptr(), d_s.data_ptr(), p.d_p.data_ptr(), n, force_c=c) == g
                if holder:
                    holder.assert_inside()
                with torch.cuda.stream(S):
                    h = digits.to("cpu", non_blocking=True)
                S.synchronize()
                got = pyref.jac_bytes_to_affine(M.combine_window_digits(cv, h.numpy().tobytes(), c, W), cv)
            st = M.last_stats()
            if holder:
                holder.__exit__(None, None, None)
        finally:
            set_stream(lib, None)
            torch.cuda.synchronize()
        assert (st["c"], st["num_windows"], st["affine_levels"] > 0) == (c, W, levels), (entry, st)
        assert got == p.want_b, (curve, n, slot, entry)


# ---------------------------------------------------------------------------------------------------------- 2. digits read at once
@pytest.mark.parametrize("slot", ["direct", "other"])
@pytest.mark.parametrize("curve,n", [("bls12_381_g1", 1 << 17), ("bls12_381_g2", 1 << 14)])
def test_digits_read_on_caller_stream_right_after_return(M, lib, spin, small, curve, n, slot):
    """The window-sharded leg's call sequence on one GPU (sharded.msm_window_sharded_device): the caller's stream set, the digits of
    this rank's window range (sharded.window_range) into a sentinel-filled device buffer, then at once, on the caller's stream, the
    copy that stands in for the all_gather and a non-blocking copy to pinned memory, and a synchronisation of that stream only. The
    digits must equal a serial call's, byte for byte, when the call ran on slot 0 and when it ran on another slot."""
    import torch
    from constantine_b200 import sharded
    p = problem(lib, curve, n)
    cv = p.cv
    c, W = M.plan(cv, n)
    g = M.digits_per_window(c)
    xyzz = 4 * cv.coord_bytes
    world = 3
    blk = -(-W // world) * g * xyzz
    serial = []
    for rank in range(world):
        wb, we = sharded.window_range(W, world, rank)
        buf = torch.zeros((we - wb) * g * xyzz, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        assert M.msm_device_digits(cv, buf.data_ptr(), p.d_sb.data_ptr(), p.d_p.data_ptr(), n, force_c=c, win_begin=wb, win_end=we) == g
        torch.cuda.synchronize()
        serial.append(buf.cpu().numpy().tobytes())
    assert pyref.jac_bytes_to_affine(M.combine_window_digits(cv, b"".join(serial), c, W), cv) == p.want_b

    S = torch.cuda.Stream()
    mine = torch.empty(blk, dtype=torch.uint8, device="cuda")
    everyone = torch.empty(world * blk, dtype=torch.uint8, device="cuda")
    h_all = torch.empty(world * blk, dtype=torch.uint8).pin_memory()
    if slot == "other":
        # grow the other slot's scratch to the whole range first: a scratch allocation frees the old buffer, which waits for the device
        whole = torch.empty(W * g * xyzz, dtype=torch.uint8, device="cuda")
        set_stream(lib, S)
        try:
            with HoldSlot0(M, spin, S, small):
                M.msm_device_digits(cv, whole.data_ptr(), p.d_sb.data_ptr(), p.d_p.data_ptr(), n, force_c=c)
        finally:
            set_stream(lib, None)
            torch.cuda.synchronize()
    got = []
    for rank in range(world):
        wb, we = sharded.window_range(W, world, rank)
        mine.fill_(SENTINEL)
        everyone.fill_(SENTINEL)
        torch.cuda.synchronize()
        set_stream(lib, S)
        try:
            holder = HoldSlot0(M, spin, S, small) if slot == "other" else None
            if holder:
                holder.__enter__()
            else:
                spin(S)
            assert M.msm_device_digits(cv, mine.data_ptr(), p.d_sb.data_ptr(), p.d_p.data_ptr(), n, force_c=c, win_begin=wb,
                                       win_end=we) == g
            if holder:
                holder.assert_inside()       # the call returned while slot 0 was still held
            with torch.cuda.stream(S):
                everyone[rank * blk:(rank + 1) * blk].copy_(mine)
                h_all.copy_(everyone, non_blocking=True)
            S.synchronize()
            if holder:
                holder.__exit__(None, None, None)
        finally:
            set_stream(lib, None)
            torch.cuda.synchronize()
        used = (we - wb) * g * xyzz
        got.append(h_all.numpy()[rank * blk:rank * blk + used].tobytes())
        assert got[-1] == serial[rank], (curve, slot, rank, "digits differ from the serial call's")
    assert pyref.jac_bytes_to_affine(M.combine_window_digits(cv, b"".join(got), c, W), cv) == p.want_b


# ---------------------------------------------------------------------------------------------------------- 3. slot reuse
@pytest.mark.parametrize("then", ["other_stream", "no_stream"])
def test_slot_reuse_after_stream_change(M, lib, spin, then):
    """A digits call on slot 0 with caller stream S1, queued behind the spin; then the caller's stream changes (to S2, whose work is
    released at the same moment as S1's, or to none) and at once a blocking MSM with other scalars runs on slot 0 again. The second
    call must not start on the slot's scratch before the digits call's work is done: both results must be right."""
    import torch
    p = problem(lib, "bls12_381_g1", 1 << 17)
    cv, n = p.cv, p.n
    c, W = M.plan(cv, n)
    g = M.digits_per_window(c)
    serial = torch.zeros(W * g * 4 * cv.coord_bytes, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    M.msm_device_digits(cv, serial.data_ptr(), p.d_sa.data_ptr(), p.d_p.data_ptr(), n, force_c=c)
    torch.cuda.synchronize()
    want_digits = serial.cpu().numpy().tobytes()
    digits = torch.full_like(serial, SENTINEL)
    S1, S2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    set_stream(lib, S1)
    try:
        spin(S1)
        released = torch.cuda.Event()
        released.record(S1)
        M.msm_device_digits(cv, digits.data_ptr(), p.d_sa.data_ptr(), p.d_p.data_ptr(), n, force_c=c)
        if then == "other_stream":
            S2.wait_event(released)
            set_stream(lib, S2)
        else:
            set_stream(lib, None)
        second = pyref.jac_bytes_to_affine(M.msm_device_ptrs(cv, p.d_sb.data_ptr(), p.d_p.data_ptr(), n, force_c=c), cv)
        S1.synchronize()
    finally:
        set_stream(lib, None)
        torch.cuda.synchronize()
    assert second == p.want_b, "the MSM after the stream change"
    got = digits.cpu().numpy().tobytes()
    assert got == want_digits, "the digits call before the stream change"
    assert pyref.jac_bytes_to_affine(M.combine_window_digits(cv, got, c, W), cv) == p.want_a


# ---------------------------------------------------------------------------------------------------------- 4. every entry family
INF48 = bytes([0xC0]) + bytes(47)


def _unhex(s):
    return bytes.fromhex(s[2:] if s.startswith("0x") else s)


def _digests(cells):
    return [hashlib.sha256(x).hexdigest() for x in cells]


class Entries:
    """Small calls of every entry family, each a zero-argument function, with its result pinned to known answers."""

    def __init__(self, M, lib):
        import torch
        g = os.path.join(ROOT, "tests", "golden")
        commit = np.load(os.path.join(g, "kzg_commit_kat.npz"))
        proof_cases = json.loads(str(np.load(os.path.join(g, "kzg_proof_kat.npz"))["cases"]))
        verify_cases = json.loads(str(np.load(os.path.join(g, "kzg_verify_kat.npz"))["cases"]))
        das = np.load(os.path.join(g, "peerdas_kat.npz"))
        das_cases = json.loads(str(das["cases"]))
        rec_cases = json.loads(str(np.load(os.path.join(g, "peerdas_recovery_kat.npz"))["cases"]))
        dver = np.load(os.path.join(g, "peerdas_verify_kat.npz"))
        dver_cases = json.loads(str(dver["cases"]))
        with open(os.path.join(g, "bls_kat.json")) as f:
            bls = json.load(f)
        blobs = [bytes(b) for b in commit["blobs"]]
        commitments = [bytes(c) for c in commit["commitments"]]

        self.ctx = ctx = M.EthKzgContext(commit["srs_lagrange_brp_compressed"].tobytes(), compressed=True)
        ctx.load_peerdas(das["srs_monomial_compressed"].tobytes())
        ctx.load_g2_setup(dver["srs_monomial_g2_compressed"].tobytes())
        cells_kat = {v["blob"]: v for v in das_cases["compute_cells_and_kzg_proofs"]["valid"]}
        self.cells = {}
        for j in range(len(blobs)):
            self.cells[j] = ctx.compute_cells(blobs[j])
            assert _digests(self.cells[j]) == cells_kat[j]["cell_sha256"], j
        self.calls, self.known = {}, {}

        # MSMs through the named symbols: 2^16 BLS12-381 G1 terms (8 MiB of input) from pinned and from pageable memory
        p = problem(lib, "bls12_381_g1", 1 << 16)
        cv = p.cv
        pin_s, pin_p = torch.from_numpy(p.sb).pin_memory(), torch.from_numpy(p.pts).pin_memory()
        tp = M.Threadpool.new(1)
        self._keep = (pin_s, pin_p, tp)
        aff = lambda b: pyref.jac_bytes_to_affine(b, cv)   # noqa: E731
        self.add("msm_pinned", lambda: aff(M.multi_scalar_mul_vartime_parallel(tp, cv, pin_s.numpy(), pin_p.numpy(), p.n)), p.want_b)
        self.add("msm_pageable", lambda: aff(M.multi_scalar_mul_vartime(cv, p.sb, p.pts, p.n)), p.want_b)
        # batches of 8 MSMs of 96 terms: host bases, and cached bases with a window table
        batch, length = 8, 96
        bsc, bpt = p.sa[:batch * length], p.pts[:batch * length]
        want_batch = [closed_form(cv, bsc[m * length:(m + 1) * length], p.k[m * length:(m + 1) * length]) for m in range(batch)]
        self.add("batch_host", lambda: [aff(r) for r in M.msm_batch(cv, bsc, bpt, batch, length)], want_batch)
        self.bases = M.CachedBases(cv, bpt, batch * length)
        assert self.bases.precompute(0, msm_len=length) >= 2
        self.add("batch_cached_table", lambda: [aff(r) for r in self.bases.msm_batch(bsc, batch, length)], want_batch)
        want_sum = pyref.ec_mul_fast(int(p.k[:5000].astype(object).sum()) % cv.fr.modulus, cv.gen, cv)
        self.add("sum_reduce", lambda: aff(M.sum_reduce_vartime(cv, p.pts[:5000])), want_sum)

        # EIP-4844
        self.add("kzg_commit", lambda: (ctx.blob_to_kzg_commitment(blobs[1]), ctx.blobs_to_kzg_commitments(blobs[:4])),
                 (commitments[1], commitments[:4]))
        pc = [c for c in proof_cases["compute_kzg_proof"]["valid"] if c["proof"] != INF48.hex()][:2]
        self.proof_blob = blobs[pc[0]["blob"]]
        bc = [c for c in proof_cases["compute_blob_kzg_proof"]["valid"] if c["proof"] != INF48.hex()][:2]
        self.add("kzg_proof", lambda: ([ctx.compute_kzg_proof(blobs[c["blob"]], bytes.fromhex(c["z"])) for c in pc],
                                       [ctx.compute_blob_kzg_proof(blobs[c["blob"]], bytes.fromhex(c["commitment"])) for c in bc]),
                 ([(bytes.fromhex(c["proof"]), bytes.fromhex(c["y"])) for c in pc], [bytes.fromhex(c["proof"]) for c in bc]))
        vk = [c for c in verify_cases["verify_kzg_proof"] if c["outcome"] in (0, 1)]
        vk = [c for c in vk if c["outcome"] == 0][:2] + [c for c in vk if c["outcome"] == 1][:2]
        vb = [c for c in verify_cases["verify_blob_kzg_proof_batch"] if c["outcome"] in (0, 1) and all(r[0] == "valid" for r in c["blobs"])]
        vb = [c for c in vb if c["outcome"] == 0][:1] + [c for c in vb if c["outcome"] == 1][:1]
        self.add("kzg_verify", lambda: ([ctx.verify_kzg_proof(*[bytes.fromhex(c[x]) for x in ("commitment", "z", "y", "proof")]) for c in vk],
                                        [ctx.verify_blob_kzg_proof_batch([blobs[r[1]] for r in c["blobs"]],
                                                                         [bytes.fromhex(x) for x in c["commitments"]],
                                                                         [bytes.fromhex(x) for x in c["proofs"]]) for c in vb]),
                 ([c["outcome"] == 0 for c in vk], [c["outcome"] == 0 for c in vb]))

        # EIP-7594
        cj = [v for v in das_cases["compute_cells_and_kzg_proofs"]["valid"] if any(x != INF48.hex() for x in v["proofs"])][0]
        self.add("das_cells", lambda: (lambda cp: (_digests(cp[0]), [x.hex() for x in cp[1]]))(ctx.compute_cells_and_kzg_proofs(blobs[cj["blob"]])),
                 (cj["cell_sha256"], cj["proofs"]))
        rc = [c for c in rec_cases["valid"] if len(c["cell_indices"]) == 64][0]
        rcells = [self.cells[v[0]][v[1]] for v in rc["cells"]]
        self.add("das_recover", lambda: (lambda cp: (_digests(cp[0]), [x.hex() for x in cp[1]]))(ctx.recover_cells_and_kzg_proofs(rc["cell_indices"], rcells)),
                 (cells_kat[rc["blob"]]["cell_sha256"], cells_kat[rc["blob"]]["proofs"]))
        dv = [c for c in dver_cases["verify"] if c["outcome"] in (0, 1) and all(isinstance(x, list) for x in c["cells"])]
        dv = [c for c in dv if c["outcome"] == 0][:2] + [c for c in dv if c["outcome"] == 1][:2]

        def das_verify():
            return [ctx.verify_cell_kzg_proof_batch([bytes.fromhex(x) for x in c["commitments"]], c["cell_indices"],
                                                    [self.cells[v[0]][v[1]] for v in c["cells"]], [bytes.fromhex(x) for x in c["proofs"]])
                    for c in dv]
        self.add("das_verify", das_verify, [c["outcome"] == 0 for c in dv])

        # BLS signatures
        bv = bls["batch_verify"]
        bv_in = [([M.eth_bls_deserialize_pubkey(_unhex(h)) for h in v["input"]["pubkeys"]], [_unhex(m) for m in v["input"]["messages"]],
                  [M.eth_bls_deserialize_signature(_unhex(h)) for h in v["input"]["signatures"]]) for v in bv]
        self.add("bls_batch_verify", lambda: [M.eth_bls_batch_verify(a, b, s, bytes(range(32))) for a, b, s in bv_in], [v["output"] for v in bv])
        av = [v for v in bls["aggregate_verify"] if v["input"]["pubkeys"]]
        av_in = []
        for v in av:
            try:
                av_in.append(([M.eth_bls_deserialize_pubkey(_unhex(h)) for h in v["input"]["pubkeys"]], [_unhex(m) for m in v["input"]["messages"]],
                              M.eth_bls_deserialize_signature(_unhex(v["input"]["signature"])), v["output"]))
            except ValueError:
                pass
        a, b, s, o = next(x for x in av_in if x[3])
        av_in.append((a, [b"another message"] + b[1:], s, False))     # the valid vector with one message changed
        assert any(o for *_, o in av_in) and not all(o for *_, o in av_in)
        self.add("bls_aggregate_verify", lambda: [M.eth_bls_aggregate_verify(a, b, s) for a, b, s, _ in av_in], [o for *_, o in av_in])
        rows, where, sets, outs = [], {}, [], []
        for v in bls["fast_aggregate_verify"]:
            try:
                pks = [M.eth_bls_deserialize_pubkey(_unhex(h)) for h in v["input"]["pubkeys"]]
                sig = M.eth_bls_deserialize_signature(_unhex(v["input"]["signature"]))
            except ValueError:
                continue
            if not pks:
                continue
            for pk in pks:
                if pk not in where:
                    where[pk] = len(rows)
                    rows.append(pk)
            sets.append(([where[pk] for pk in pks], _unhex(v["input"]["message"]), sig))
            outs.append(v["output"])
        idx, _, sig = next(s for s, o in zip(sets, outs) if o)
        sets.append((idx, b"another message", sig))                  # a valid set with its message changed
        outs.append(False)
        assert any(outs) and not all(outs)
        self.registry = M.CachedBases("bls12_381_g1", b"".join(rows))
        self.sets, self.set_statuses = sets, [0 if o else 1 for o in outs]
        good = [s for s, o in zip(sets, outs) if o]
        self.add("bls_sets", lambda: (M.eth_bls_verify_sets(self.registry, sets), M.eth_bls_batch_verify_sets(self.registry, good, bytes(range(32))),
                                      M.eth_bls_batch_verify_sets(self.registry, sets, bytes(range(32)))),
                 ([0 if o else 1 for o in outs], True, False))
        g1_raw = [_unhex(v["input"]["pubkey"]) for v in bls["deserialization_G1"] if v["status"] != "length"]
        g2_raw = [_unhex(v["input"]["signature"]) for v in bls["deserialization_G2"] if v["status"] != "length"]

        def single(fn, raw, size):
            try:
                return fn(raw), 0
            except ValueError as e:
                return bytes(size), e.args[0]
        want_g1 = [single(M.eth_bls_deserialize_pubkey, b, 96) for b in g1_raw]
        want_g2 = [single(M.eth_bls_deserialize_signature, b, 192) for b in g2_raw]
        assert any(s for _, s in want_g1) and any(s == 0 for _, s in want_g1)
        self.add("bls_decode", lambda: (M.eth_bls_deserialize_pubkeys(g1_raw * 5), M.eth_bls_deserialize_signatures(g2_raw * 3)),
                 (tuple(list(x) for x in zip(*(want_g1 * 5))), tuple(list(x) for x in zip(*(want_g2 * 3)))))

        # every known answer holds without a caller's stream, single-threaded
        for name in self.calls:
            got = self.call(name)
            assert got == self.known[name], name

    def add(self, name, fn, known):
        self.calls[name], self.known[name] = fn, known

    def call(self, name):
        return self.calls[name]()

    def close(self):
        self.bases.free()
        self.registry.free()
        self.ctx.delete()
        self._keep[2].shutdown()


@pytest.fixture(scope="module")
def entries(M, lib):
    e = Entries(M, lib)
    yield e
    e.close()


@pytest.mark.parametrize("slot", ["direct", "other"])
def test_every_entry_family_under_caller_stream(M, lib, spin, small, entries, slot):
    """Named MSM symbols (pinned and pageable input), batches (host bases, cached bases with a window table), sum_reduce, KZG commit /
    proof / verify, PeerDAS cells / recovery / verification, BLS batch_verify / aggregate_verify / sets / batched decode: the same
    bytes with the caller's stream set as without, on slot 0 and (while a helper holds slot 0) on another slot."""
    import torch
    S = torch.cuda.Stream()
    set_stream(lib, S)
    try:
        for name in entries.calls:
            if slot == "other":
                with HoldSlot0(M, spin, S, small) as holder:
                    holder.assert_inside()
                    got = entries.call(name)
            else:
                got = entries.call(name)
            assert got == entries.known[name], (name, slot)
    finally:
        set_stream(lib, None)
        torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- 5. concurrent callers
@pytest.mark.parametrize("with_stream", [False, True])
@pytest.mark.parametrize("slots", [1, 2, 4])
def test_concurrent_callers_across_entries(M, lib, entries, slots, with_stream):
    """8 threads, each with its own mix of the entries above on one shared EthKzgContext and one registry, against the single-threaded
    results. Each thread also makes an MSM of its own length and checks that last_stats() shows that call's window size and phase
    times, and checks EthKzgContext.last_timing and eth_bls_last_timing right after its own calls: the statistics are per thread."""
    import torch
    p = problem(lib, "bls12_381_g1", 1 << 16)
    cv = p.cv
    names = list(entries.calls)
    lengths = [1 << (6 + t) for t in range(8)]
    prefix = {}
    acc = 0
    for i in range(p.n):
        acc += int.from_bytes(p.sb[i].tobytes(), "little") * int(p.k[i])
        if i + 1 in lengths:
            prefix[i + 1] = pyref.ec_mul_fast(acc % cv.fr.modulus, cv.gen, cv)
    errors = []
    start = threading.Barrier(8)

    def worker(t):
        try:
            rnd = random.Random(slots * 100 + t)
            mix = [names[(t + 3 * j) % len(names)] for j in range(4)]
            rnd.shuffle(mix)
            start.wait()
            for name in mix:
                got = entries.call(name)
                if got != entries.known[name]:
                    errors.append((t, name))
                n = lengths[t]
                r = M.multi_scalar_mul_vartime(cv, p.sb[:n], p.pts[:n], n)
                st = M.last_stats()
                c, W = M.plan(cv, n)
                if pyref.jac_bytes_to_affine(r, cv) != prefix[n]:
                    errors.append((t, "msm", n))
                if (st["c"], st["num_windows"]) != (c, W) or not (st["ms_total"] > 0 and st["ms_sort"] > 0 and st["ms_reduce"] > 0):
                    errors.append((t, "last_stats", n, st))
            if t % 2:
                entries.ctx.compute_kzg_proof(entries.proof_blob, (12345 + t).to_bytes(32, "big"))
                tm = entries.ctx.last_timing()
                if not (tm["ms_host"] > 0 and tm["ms_quotient"] > 0):
                    errors.append((t, "kzg last_timing", tm))
            else:
                # verify_sets runs no G2 MSM (ms_msm == 0), batch_verify does: another thread's call must not show through
                verify_sets = t % 4 == 0
                if verify_sets:
                    if M.eth_bls_verify_sets(entries.registry, entries.sets) != entries.set_statuses:
                        errors.append((t, "verify_sets"))
                else:
                    entries.call("bls_batch_verify")
                tm = M.eth_bls_last_timing()
                if not tm["ms_final"] > 0 or (tm["ms_msm"] == 0) != verify_sets:
                    errors.append((t, "bls last_timing", verify_sets, tm))
        except Exception as e:        # noqa: BLE001 -- reported by the main thread
            errors.append((t, repr(e)))

    lib.ctt_b200_set_concurrency(slots)
    S = torch.cuda.Stream() if with_stream else None
    set_stream(lib, S)
    try:
        threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
    finally:
        set_stream(lib, None)
        lib.ctt_b200_set_concurrency(2)
        torch.cuda.synchronize()
    assert not errors, errors
