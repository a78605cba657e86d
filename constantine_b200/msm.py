"""Host-side mirror of the reference's MSM interface on top of the C ABI.

Names follow the reference:
  multi_scalar_mul_vartime_parallel  <->  reference constantine/math/elliptic/ec_multi_scalar_mul_parallel.nim:588-628
      (`tp.multiScalarMul_vartime_parallel(r, coefs, points, len)`, BigInt and Fr overloads), exported to C as
      ctt_<curve>_<jac|prj>_multi_scalar_mul_<big|fr>_coefs_vartime_parallel (bindings/c_curve_decls_parallel.nim:31-45)
  multi_scalar_mul_vartime           <->  reference constantine/math/elliptic/ec_multi_scalar_mul.nim:525-568 (serial twin)
  Threadpool                          <->  reference constantine/threadpool/threadpool.nim:943-1041 (new / shutdown)
  PrecomputedMSM (init / msm_vartime) <->  reference constantine/math/elliptic/ec_multi_scalar_mul_precomp.nim:28-33, 109-161, 192-240
  PrecomputedMSMBank                  <->  the `openArray[PrecomputedMSM]` banks of reference constantine/math/matrix/toeplitz.nim:347-360
  sum_reduce_vartime(_parallel)       <->  reference constantine/math/elliptic/ec_shortweierstrass_batch_ops.nim:649-664,
                                           ec_shortweierstrass_batch_ops_parallel.nim:110-123

Buffers are `bytes`/`bytearray`/numpy arrays/anything exposing the buffer protocol, laid out exactly like the
reference's C structs (see include/ctt_b200_msm.h). Results come back as `bytes` of the _jac / _prj struct.
Every call goes through the named extern "C" symbol -- this module adds no arithmetic.
"""
import ctypes
import operator

from . import _lib
from .curves import CURVES, CurveParams

OUT_JAC, OUT_PRJ, OUT_XYZZ = 0, 1, 2


def _curve(curve) -> CurveParams:
    return curve if isinstance(curve, CurveParams) else CURVES[curve]


def _buf(b):
    """ctypes view of a read-only buffer without copying when possible."""
    if isinstance(b, (bytes, bytearray)):
        return (ctypes.c_char * len(b)).from_buffer_copy(b) if isinstance(b, bytes) else (ctypes.c_char * len(b)).from_buffer(b)
    mv = memoryview(b).cast("B")
    if mv.readonly:
        return (ctypes.c_char * len(mv)).from_buffer_copy(mv)
    return (ctypes.c_char * len(mv)).from_buffer(mv)


class Threadpool:
    """Opaque handle kept for source compatibility with reference callers (`Threadpool.new(n)` / `shutdown`)."""

    def __init__(self, num_threads: int = 0):
        lib = _lib.load()
        self._h = lib.ctt_threadpool_new(num_threads or lib.ctt_cpu_get_num_threads_os())

    @classmethod
    def new(cls, num_threads: int = 0):
        return cls(num_threads)

    def shutdown(self):
        if self._h:
            _lib.load().ctt_threadpool_shutdown(self._h)
            self._h = None


def set_devices(device_ids) -> None:
    """Spread every host-pointer MSM of this process over these CUDA devices (ctt_b200_set_devices; [] = caller's device only)."""
    ids = list(device_ids)
    arr = (ctypes.c_int * max(1, len(ids)))(*ids)
    if _lib.load().ctt_b200_set_devices(arr, len(ids)) != 0:
        raise ValueError(f"unknown CUDA device in {ids}")


def device_count() -> int:
    return _lib.load().ctt_b200_device_count()


def _symbol(curve: CurveParams, out: str, coef_kind: str, parallel: bool) -> str:
    return f"ctt_{curve.cprefix}_{out}_multi_scalar_mul_{coef_kind}_coefs_vartime" + ("_parallel" if parallel else "")


def multi_scalar_mul_vartime_parallel(tp, curve, coefs, points, length=None, out="jac", coef_kind="big") -> bytes:
    """r <- [a0]P0 + ... + [a_{n-1}]P_{n-1}  through ctt_<curve>_<out>_multi_scalar_mul_<coef_kind>_coefs_vartime_parallel.

    coefs: n x 32 bytes (canonical BigInt for coef_kind="big", Fr Montgomery residues for "fr");
    points: n affine structs. Returns the _jac / _prj struct bytes.
    """
    cv = _curve(curve)
    n = length if length is not None else len(memoryview(points).cast("B")) // cv.aff_bytes
    fn = _lib.named_msm(_symbol(cv, out, coef_kind, True))
    r = ctypes.create_string_buffer(cv.jac_bytes)
    cb, pb = _buf(coefs), _buf(points)
    fn(getattr(tp, "_h", None), r, cb, pb, n)
    return r.raw


def multi_scalar_mul_vartime(curve, coefs, points, length=None, out="jac", coef_kind="big") -> bytes:
    cv = _curve(curve)
    n = length if length is not None else len(memoryview(points).cast("B")) // cv.aff_bytes
    fn = _lib.named_msm(_symbol(cv, out, coef_kind, False))
    r = ctypes.create_string_buffer(cv.jac_bytes)
    cb, pb = _buf(coefs), _buf(points)
    fn(r, cb, pb, n)
    return r.raw


def msm_device_ptrs(curve, d_coefs: int, d_points: int, n: int, out=OUT_JAC, fr_mont=False, force_c=0,
                    win_begin=0, win_end=-1) -> bytes:
    """MSM over device-resident inputs (raw device pointers, e.g. torch tensor .data_ptr())."""
    cv = _curve(curve)
    size = cv.coord_bytes * (4 if out == OUT_XYZZ else 3)
    r = ctypes.create_string_buffer(size)
    rc = _lib.load().ctt_b200_msm_device(cv.curve_id, out, r, d_coefs, d_points, n, int(fr_mont), force_c, win_begin, win_end)
    if rc != 0:
        raise ValueError("ctt_b200_msm_device: bad curve id")
    return r.raw


def digits_per_window(c: int) -> int:
    """radix-16 digits of a window sum (k_plane_combine): ceil((c - 1) / 4)."""
    return (c - 1 + 3) // 4


def msm_device_digits(curve, d_digits_out: int, d_coefs: int, d_points: int, n: int, fr_mont=False, force_c=0, win_begin=0, win_end=-1) -> int:
    """Window range [win_begin, win_end) of an MSM over device-resident inputs; the radix-16 digits of the window sums stay in the
    device buffer d_digits_out (raw XYZZ, window-major). NOT synchronised: work queued afterwards on the caller's stream
    (ctt_b200_set_stream) sees the digits; without a caller's stream, synchronise the device before reading them."""
    cv = _curve(curve)
    g = _lib.load().ctt_b200_msm_device_digits(cv.curve_id, d_digits_out, d_coefs, d_points, n, int(fr_mont), force_c, win_begin, win_end)
    if g < 0:
        raise ValueError("ctt_b200_msm_device_digits failed")
    return g


def combine_window_digits(curve, h_digits, c: int, num_windows: int, out=OUT_JAC) -> bytes:
    """digits of all windows 0..num_windows-1 (host buffer, window-major, digits_per_window(c) XYZZ points each) -> result struct."""
    cv = _curve(curve)
    r = ctypes.create_string_buffer(cv.coord_bytes * (4 if out == OUT_XYZZ else 3))
    if _lib.load().ctt_b200_combine_window_digits(cv.curve_id, out, r, _buf(h_digits), c, num_windows) != 0:
        raise ValueError("ctt_b200_combine_window_digits failed")
    return r.raw


def sum_partials(curve, partials: bytes, count: int, out=OUT_JAC) -> bytes:
    cv = _curve(curve)
    size = cv.coord_bytes * (4 if out == OUT_XYZZ else 3)
    r = ctypes.create_string_buffer(size)
    rc = _lib.load().ctt_b200_sum_partials(cv.curve_id, out, r, _buf(partials), count)
    if rc != 0:
        raise ValueError("ctt_b200_sum_partials: bad curve id")
    return r.raw


def plan(curve, n: int, force_c: int = 0):
    cv = _curve(curve)
    c, w = ctypes.c_int(0), ctypes.c_int(0)
    _lib.load().ctt_b200_plan(cv.curve_id, n, force_c, ctypes.byref(c), ctypes.byref(w))
    return c.value, w.value


def last_stats() -> dict:
    s = _lib.Stats()
    _lib.load().ctt_b200_last_stats(ctypes.byref(s))
    return {k: getattr(s, k) for k, _ in s._fields_}


class CachedBases:
    """Device-resident bases (reference constantine-rust/constantine-halo2-zal/src/lib.rs:58-95 caching hooks)."""

    def __init__(self, curve, points, length=None):
        self.curve = _curve(curve)
        self.n = length if length is not None else len(memoryview(points).cast("B")) // self.curve.aff_bytes
        self._h = _lib.load().ctt_b200_bases_upload(self.curve.curve_id, _buf(points), self.n)

    @classmethod
    def _from_handle(cls, curve, handle, n):
        """Wrap a ctt_b200_bases handle that a C entry made (eth_bls_registry_from_compressed); free() releases it."""
        self = cls.__new__(cls)
        self.curve, self.n, self._h = _curve(curve), n, handle
        return self

    def precompute(self, c: int = 0, msm_len: int = 0) -> int:
        """One-time table of window multiples 2^(c w) P_i (ctt_b200_bases_precompute[_for]); returns the window size
        used. msm_len: length of the MSMs the bases will serve when they hold a whole bank (default: all bases)."""
        lib = _lib.load()
        rc = lib.ctt_b200_bases_precompute_for(self._h, msm_len, c) if msm_len else lib.ctt_b200_bases_precompute(self._h, c)
        if rc < 0:
            raise ValueError("ctt_b200_bases_precompute failed")
        return rc

    def msm_batch(self, coefs, batch: int, length: int, out=OUT_JAC, coef_kind="big", shared_points=False) -> list:
        """`batch` MSMs of `length` terms in one engine pass over the cached bases (ctt_b200_msm_batch_cached_bases)."""
        size = self.curve.coord_bytes * (4 if out == OUT_XYZZ else 3)
        r = ctypes.create_string_buffer(max(1, size * batch))
        rc = _lib.load().ctt_b200_msm_batch_cached_bases(self._h, out, r, _buf(coefs), batch, length, int(coef_kind == "fr"),
                                                         int(shared_points))
        if rc != 0:
            raise ValueError("ctt_b200_msm_batch_cached_bases failed (batch*len exceeds the cached bases?)")
        return [r.raw[m * size:(m + 1) * size] for m in range(batch)]

    def msm(self, coefs, length=None, out=OUT_JAC, coef_kind="big") -> bytes:
        n = length if length is not None else len(memoryview(coefs).cast("B")) // 32
        if out not in (OUT_JAC, OUT_PRJ, OUT_XYZZ):
            raise ValueError("out must be OUT_JAC, OUT_PRJ or OUT_XYZZ")
        r = ctypes.create_string_buffer(self.curve.coord_bytes * (4 if out == OUT_XYZZ else 3))
        rc = _lib.load().ctt_b200_msm_cached_bases(self._h, out, r, _buf(coefs), n, int(coef_kind == "fr"))
        if rc != 0:
            raise ValueError("ctt_b200_msm_cached_bases failed (len exceeds the cached bases?)")
        return r.raw

    def free(self):
        if self._h:
            _lib.load().ctt_b200_bases_free(self._h)
            self._h = None


FFT_KINDS = {"fft_nn": 0, "fft_nr": 1, "ifft_nn": 2, "ifft_rn": 3,
             "coset_fft_nn": 4, "coset_fft_nr": 5, "coset_ifft_nn": 6, "coset_ifft_rn": 7}
FFT_FIELDS = {"bls12_381": 0, "bn254_snarks": 1, "pallas": 2, "vesta": 3}


class FFTError(ValueError):
    """A non-zero status of the FFT entries: 2 too many values, 3 size not a power of two, 4 omega not of the domain's order,
    5 bad argument (the numbering of the reference's FFTStatus for 1..3)."""

    def __init__(self, status: int, what: str):
        super().__init__(f"{what}: status {status}")
        self.status = status


def _fft_field_id(curve) -> int:
    if isinstance(curve, int):
        return curve
    if isinstance(curve, CurveParams):
        curve = curve.name
    if curve in FFT_FIELDS:
        return FFT_FIELDS[curve]
    return _curve(curve).curve_id


def _fr_struct(x) -> bytes:
    """An Fr struct (Montgomery, 4 x u64): 32 bytes as given, or an int already in Montgomery form."""
    if isinstance(x, int):
        return x.to_bytes(32, "little")
    b = bytes(memoryview(x).cast("B"))
    if len(b) != 32:
        raise ValueError("an Fr struct is 32 bytes")
    return b


class FFTDomain:
    """The reference's FrFFT_Descriptor (constantine/math/polynomials/fft_fields.nim) on the device: the Fr of `curve` (curve id
    0..3 or its name), order 2^log_order, generator `omega` (32-byte Fr struct, Montgomery form) of exactly that order. One domain
    serves every power-of-two length n <= 2^log_order with omega^(2^log_order / n). Values are reduced Montgomery residues: bytes
    of batch * n * 32, or numpy uint64[batch * n, 4]; results come back in the same type. `batch` transforms lie back to back."""

    def __init__(self, curve, omega, log_order: int):
        st = ctypes.c_int(0)
        self.field_id, self.log_order = _fft_field_id(curve), log_order
        self._h = _lib.load().ctt_b200_fft_domain_new(self.field_id, _fr_struct(omega), log_order, ctypes.byref(st))
        if not self._h:
            raise FFTError(st.value, "ctt_b200_fft_domain_new")

    def _run(self, kind: str, vals, batch: int, shift):
        lib = _lib.load()
        sh = _fr_struct(shift) if shift is not None else None
        is_np = type(vals).__module__ == "numpy"
        if is_np:
            # the caller's array is read in place and the result written straight into a new array: no intermediate copies
            import numpy as np
            a = np.ascontiguousarray(vals, dtype=np.uint64).reshape(-1, 4)
            out = np.empty_like(a)
            src, dst, total = a.ctypes.data, out.ctypes.data, len(a)
        else:
            src = _buf(vals)
            total = len(src) // 32
            out = ctypes.create_string_buffer(max(1, 32 * total))
            dst = out
        if batch < 1 or total % batch:
            raise ValueError("the values are not batch transforms of one length")
        rc = lib.ctt_b200_fft(self._h, FFT_KINDS[kind], dst, src if total else dst, total // batch, batch, sh)
        if rc != 0:
            raise FFTError(rc, kind)
        return out if is_np else out.raw[:32 * total]

    def _run_device(self, kind: str, d_out: int, d_in: int, n: int, batch: int, shift):
        sh = _fr_struct(shift) if shift is not None else None
        rc = _lib.load().ctt_b200_fft_device(self._h, FFT_KINDS[kind], d_out, d_in, n, batch, sh)
        if rc != 0:
            raise FFTError(rc, kind + "_device")

    def fft_nn(self, vals, batch=1): return self._run("fft_nn", vals, batch, None)
    def fft_nr(self, vals, batch=1): return self._run("fft_nr", vals, batch, None)
    def ifft_nn(self, vals, batch=1): return self._run("ifft_nn", vals, batch, None)
    def ifft_rn(self, vals, batch=1): return self._run("ifft_rn", vals, batch, None)
    def coset_fft_nn(self, vals, shift, batch=1): return self._run("coset_fft_nn", vals, batch, shift)
    def coset_fft_nr(self, vals, shift, batch=1): return self._run("coset_fft_nr", vals, batch, shift)
    def coset_ifft_nn(self, vals, shift, batch=1): return self._run("coset_ifft_nn", vals, batch, shift)
    def coset_ifft_rn(self, vals, shift, batch=1): return self._run("coset_ifft_rn", vals, batch, shift)

    # device pointers (e.g. a torch tensor's data_ptr()); the stream contract of ctt_b200_fft_device
    def fft_nn_device(self, d_out, d_in, n, batch=1): self._run_device("fft_nn", d_out, d_in, n, batch, None)
    def fft_nr_device(self, d_out, d_in, n, batch=1): self._run_device("fft_nr", d_out, d_in, n, batch, None)
    def ifft_nn_device(self, d_out, d_in, n, batch=1): self._run_device("ifft_nn", d_out, d_in, n, batch, None)
    def ifft_rn_device(self, d_out, d_in, n, batch=1): self._run_device("ifft_rn", d_out, d_in, n, batch, None)
    def coset_fft_nn_device(self, d_out, d_in, n, shift, batch=1): self._run_device("coset_fft_nn", d_out, d_in, n, batch, shift)
    def coset_fft_nr_device(self, d_out, d_in, n, shift, batch=1): self._run_device("coset_fft_nr", d_out, d_in, n, batch, shift)
    def coset_ifft_nn_device(self, d_out, d_in, n, shift, batch=1): self._run_device("coset_ifft_nn", d_out, d_in, n, batch, shift)
    def coset_ifft_rn_device(self, d_out, d_in, n, shift, batch=1): self._run_device("coset_ifft_rn", d_out, d_in, n, batch, shift)

    @staticmethod
    def last_timing() -> dict:
        """The calling thread's last FFT call (ms): upload, kernels and copy back (device entry: kernels only)."""
        v = [ctypes.c_float() for _ in range(3)]
        _lib.load().ctt_b200_fft_last_timing(*[ctypes.byref(x) for x in v])
        return dict(zip(("ms_h2d", "ms_kernels", "ms_d2h"), (x.value for x in v)))

    def free(self):
        if self._h:
            _lib.load().ctt_b200_fft_domain_free(self._h)
            self._h = None


def msm_batch(curve, coefs, points, batch: int, length: int, out=OUT_JAC, coef_kind="big", shared_points=False) -> list:
    """r[m] = sum_i coefs[m*length + i] * points[(0 if shared_points else m*length) + i] for m < batch, host buffers, one
    engine pass (ctt_b200_msm_batch_host). Returns the list of result structs."""
    cv = _curve(curve)
    size = cv.coord_bytes * (4 if out == OUT_XYZZ else 3)
    r = ctypes.create_string_buffer(max(1, size * batch))
    rc = _lib.load().ctt_b200_msm_batch_host(cv.curve_id, out, r, _buf(coefs), _buf(points), batch, length, int(coef_kind == "fr"),
                                             int(shared_points))
    if rc != 0:
        raise ValueError("ctt_b200_msm_batch_host: bad curve id")
    return [r.raw[m * size:(m + 1) * size] for m in range(batch)]


class PrecomputedMSM:
    """Fixed-base MSM context, the reference's `PrecomputedMSM[EC, N]`.

    reference: `ctx.init(basis, t, b)` builds comb tables (stride t, window b) on the host and `ctx.msm_vartime(r, scalars)`
    walks them with mixed additions. Here `init` uploads the basis and builds the table 2^(c w) P_i in HBM and
    `msm_vartime` is one engine pass with a single bucket set. (t, b) are accepted for source compatibility; they
    parametrise the reference's table shape, not the result -- the window c plays their role and is chosen by the
    engine unless given.
    """

    def __init__(self):
        self._bases = None
        self.N = 0

    def init(self, curve, basis, t: int = 0, b: int = 0, c: int = 0):
        self._bases = CachedBases(curve, basis)
        self.N = self._bases.n
        self.c = self._bases.precompute(c)
        return self

    def msm_vartime(self, scalars, out="jac", coef_kind="big") -> bytes:
        n = len(memoryview(scalars).cast("B")) // 32
        if n != self.N:
            raise ValueError("PrecomputedMSM.msm_vartime: need exactly N scalars")     # reference: openArray of length N
        return self._bases.msm(scalars, n, OUT_JAC if out == "jac" else OUT_PRJ, coef_kind)

    def free(self):
        if self._bases:
            self._bases.free()
            self._bases = None


class PrecomputedMSMBank:
    """`count` PrecomputedMSM objects of N points each, evaluated together (the reference loops over the bank,
    matrix/toeplitz.nim:357-360: `polyphaseSpectrumBank[i].msm_vartime(output[i], scalars_i)`)."""

    def __init__(self, curve, bases, count: int, n: int, c: int = 0):
        self.count, self.N = count, n
        self._bases = CachedBases(curve, bases, count * n)
        self.c = self._bases.precompute(c, msm_len=n)

    def msm_vartime(self, scalars, out="jac", coef_kind="big") -> list:
        return self._bases.msm_batch(scalars, self.count, self.N, OUT_JAC if out == "jac" else OUT_PRJ, coef_kind)

    def free(self):
        self._bases.free()


def sum_reduce_vartime(curve, points, length=None, out="jac") -> bytes:
    """r = P_0 + ... + P_{n-1} (ctt_b200_sum_reduce_host)."""
    cv = _curve(curve)
    n = length if length is not None else len(memoryview(points).cast("B")) // cv.aff_bytes
    r = ctypes.create_string_buffer(cv.jac_bytes)
    rc = _lib.load().ctt_b200_sum_reduce_host(cv.curve_id, OUT_JAC if out == "jac" else OUT_PRJ, r, _buf(points), n)
    if rc != 0:
        raise ValueError("ctt_b200_sum_reduce_host: bad curve id")
    return r.raw


def sum_reduce_vartime_parallel(tp, curve, points, length=None, out="jac") -> bytes:
    return sum_reduce_vartime(curve, points, length, out)


EVM_STATUS = ("cttEVM_Success", "cttEVM_InvalidInputSize", "cttEVM_InvalidOutputSize", "cttEVM_IntLargerThanModulus",
              "cttEVM_PointNotOnCurve", "cttEVM_PointNotInSubgroup", "cttEVM_VerificationFailure", "cttEVM_MalformedSignature")


def eth_evm_bls12381_g1msm(inputs: bytes, out_len: int = 128):
    """EIP-2537 BLS12_G1MSM through ctt_eth_evm_bls12381_g1msm (reference constantine/ethereum_evm_precompiles.nim:894-975).
    Returns (status name, output bytes)."""
    r = ctypes.create_string_buffer(out_len)
    st = _lib.load().ctt_eth_evm_bls12381_g1msm(r, out_len, bytes(inputs), len(inputs))
    return EVM_STATUS[st], r.raw


def eth_evm_bls12381_g2msm(inputs: bytes, out_len: int = 256):
    """EIP-2537 BLS12_G2MSM through ctt_eth_evm_bls12381_g2msm (reference constantine/ethereum_evm_precompiles.nim:977-1060)."""
    r = ctypes.create_string_buffer(out_len)
    st = _lib.load().ctt_eth_evm_bls12381_g2msm(r, out_len, bytes(inputs), len(inputs))
    return EVM_STATUS[st], r.raw


def eth_evm_bn254_ecpairingcheck(inputs: bytes, out_len: int = 32):
    """EIP-197 ecPairing on BN254 through ctt_eth_evm_bn254_ecpairingcheck (reference constantine/ethereum_evm_precompiles.nim:543-626):
    k x 192 bytes of (P.x, P.y, Q.x_im, Q.x_re, Q.y_im, Q.y_re), 32-byte big-endian each. Returns (status name, output bytes), the
    output 32 bytes holding 0 or 1. A pair with an infinity point contributes 1 and the other pairs still count (EIP-197)."""
    r = ctypes.create_string_buffer(max(out_len, 1))
    inputs = bytes(inputs)
    st = _lib.load().ctt_eth_evm_bn254_ecpairingcheck(r, out_len, inputs, len(inputs))
    return EVM_STATUS[st], r.raw[:out_len]


def _eth_evm_pairingcheck_batch(name, calls) -> list:
    """Many independent pairing-check calls in one pass through the offsets-based batch entry `name`."""
    calls = [bytes(c) for c in calls]
    k = len(calls)
    if k == 0:
        return []
    offsets = (ctypes.c_size_t * (k + 1))()
    for i, c in enumerate(calls):
        offsets[i + 1] = offsets[i] + len(c)
    data = b"".join(calls) or b"\0"
    r = ctypes.create_string_buffer(32 * k)
    statuses = ctypes.create_string_buffer(k)
    st = getattr(_lib.load(), name)(r, statuses, data, offsets[k], offsets, k)
    if st != 0:
        raise ValueError(EVM_STATUS[st])
    raw = r.raw
    return [(EVM_STATUS[statuses.raw[i]], raw[32 * i:32 * i + 32]) for i in range(k)]


def _eth_evm_records_batch(name, data, in_bytes, out_bytes):
    """n fixed-size records of in_bytes in one pass through the batch entry `name`: ([status name] * n, n x out_bytes)."""
    data = bytes(data)
    if len(data) % in_bytes:
        raise ValueError("inputs must be a multiple of %d bytes" % in_bytes)
    n = len(data) // in_bytes
    r = ctypes.create_string_buffer(max(out_bytes * n, 1))
    statuses = ctypes.create_string_buffer(max(n, 1))
    st = getattr(_lib.load(), name)(r, statuses, data or b"\0", n)
    if st != 0:
        raise ValueError(EVM_STATUS[st])
    return [EVM_STATUS[b] for b in statuses.raw[:n]], r.raw[:out_bytes * n]


def eth_evm_bn254_ecpairingcheck_batch(calls) -> list:
    """Many independent ecPairing calls in one pass (ctt_b200_eth_evm_bn254_ecpairingcheck_batch): calls is a sequence of byte
    strings; returns [(status name, 32 output bytes)] in the same order, as the single entry gives them per call."""
    return _eth_evm_pairingcheck_batch("ctt_b200_eth_evm_bn254_ecpairingcheck_batch", calls)


def eth_evm_bn254_last_timing() -> dict:
    """Host checks and packing, device decoding, Miller loops, and products with final exponentiations (ms) of the calling thread's
    last ecPairing call."""
    v = [ctypes.c_float(0) for _ in range(4)]
    _lib.load().ctt_b200_eth_evm_bn254_last_timing(*[ctypes.byref(x) for x in v])
    return dict(zip(("ms_host", "ms_decode", "ms_miller", "ms_final"), (x.value for x in v)))


def eth_evm_bls12381_pairingcheck(inputs: bytes, out_len: int = 32):
    """EIP-2537 BLS12_PAIRING_CHECK through ctt_eth_evm_bls12381_pairingcheck (reference constantine/ethereum_evm_precompiles.nim:
    1064-1125): k x 384 bytes of (P.x, P.y, Q.x.c0, Q.x.c1, Q.y.c0, Q.y.c1), 64-byte big-endian each. Returns (status name, output
    bytes), the output 32 bytes holding 0 or 1 (zeros when the call fails). The empty call is cttEVM_InvalidInputSize."""
    r = ctypes.create_string_buffer(max(out_len, 1))
    inputs = bytes(inputs)
    st = _lib.load().ctt_eth_evm_bls12381_pairingcheck(r, out_len, inputs, len(inputs))
    return EVM_STATUS[st], r.raw[:out_len]


def eth_evm_bls12381_pairingcheck_batch(calls) -> list:
    """Many independent BLS12_PAIRING_CHECK calls in one pass (ctt_b200_eth_evm_bls12381_pairingcheck_batch): calls is a sequence of
    byte strings; returns [(status name, 32 output bytes)] in the same order, as the single entry gives them per call."""
    return _eth_evm_pairingcheck_batch("ctt_b200_eth_evm_bls12381_pairingcheck_batch", calls)


def _eth_evm_bls12381_map(name, inputs, out_len):
    r = ctypes.create_string_buffer(max(out_len, 1))
    inputs = bytes(inputs)
    st = getattr(_lib.load(), name)(r, out_len, inputs, len(inputs))
    return EVM_STATUS[st], r.raw[:out_len]


def eth_evm_bls12381_map_fp_to_g1(inputs: bytes, out_len: int = 128):
    """EIP-2537 BLS12_MAP_FP_TO_G1 through ctt_eth_evm_bls12381_map_fp_to_g1: u (64 bytes) -> (status name, the affine G1 point,
    128 bytes; zeros for infinity)."""
    return _eth_evm_bls12381_map("ctt_eth_evm_bls12381_map_fp_to_g1", inputs, out_len)


def eth_evm_bls12381_map_fp2_to_g2(inputs: bytes, out_len: int = 256):
    """EIP-2537 BLS12_MAP_FP2_TO_G2 through ctt_eth_evm_bls12381_map_fp2_to_g2: u = (c0, c1) (128 bytes) -> (status name, the affine
    G2 point, 256 bytes; zeros for infinity)."""
    return _eth_evm_bls12381_map("ctt_eth_evm_bls12381_map_fp2_to_g2", inputs, out_len)


def eth_evm_bls12381_map_fp_to_g1_batch(data: bytes):
    """n maps to G1 in one pass (ctt_b200_eth_evm_bls12381_map_fp_to_g1_batch): data is n x 64 bytes; returns ([status name] * n,
    n x 128 output bytes), a failed element's output zeros."""
    return _eth_evm_records_batch("ctt_b200_eth_evm_bls12381_map_fp_to_g1_batch", data, 64, 128)


def eth_evm_bls12381_map_fp2_to_g2_batch(data: bytes):
    """n maps to G2 in one pass (ctt_b200_eth_evm_bls12381_map_fp2_to_g2_batch): data is n x 128 bytes; returns ([status name] * n,
    n x 256 output bytes), a failed element's output zeros."""
    return _eth_evm_records_batch("ctt_b200_eth_evm_bls12381_map_fp2_to_g2_batch", data, 128, 256)


def eth_evm_bls12381_last_timing() -> dict:
    """Host checks and packing, device pair decoding, maps, Miller loops, and products with final exponentiations (ms) of the calling
    thread's last EIP-2537 pairing-check or map call; phases the call does not have read 0."""
    v = [ctypes.c_float(0) for _ in range(5)]
    _lib.load().ctt_b200_eth_evm_bls12381_last_timing(*[ctypes.byref(x) for x in v])
    return dict(zip(("ms_host", "ms_decode", "ms_map", "ms_miller", "ms_final"), (x.value for x in v)))


# EVM curve operations: name -> (record bytes of a batch, output bytes)
ECOPS = {"bn254_g1add": (128, 64), "bn254_g1mul": (96, 64), "bls12381_g1add": (256, 128), "bls12381_g2add": (512, 256),
         "bls12381_g1mul": (160, 128), "bls12381_g2mul": (288, 256)}


def _eth_evm_ecop(name, inputs, out_len):
    r = ctypes.create_string_buffer(max(out_len, 1))
    inputs = bytes(inputs)
    st = getattr(_lib.load(), "ctt_eth_evm_" + name)(r, out_len, inputs, len(inputs))
    return EVM_STATUS[st], r.raw[:out_len]


def eth_evm_bn254_g1add(inputs: bytes, out_len: int = 64):
    """EIP-196 ECADD through ctt_eth_evm_bn254_g1add: P, Q (32-byte big-endian coordinates; the input zero-padded or truncated to
    128 bytes) -> (status name, P + Q affine, 64 bytes; zeros for infinity)."""
    return _eth_evm_ecop("bn254_g1add", inputs, out_len)


def eth_evm_bn254_g1mul(inputs: bytes, out_len: int = 64):
    """EIP-196 ECMUL through ctt_eth_evm_bn254_g1mul: P and a 32-byte scalar (padded or truncated to 96 bytes) -> (status name,
    [s]P affine, 64 bytes)."""
    return _eth_evm_ecop("bn254_g1mul", inputs, out_len)


def eth_evm_bls12381_g1add(inputs: bytes, out_len: int = 128):
    """EIP-2537 BLS12_G1ADD through ctt_eth_evm_bls12381_g1add: P, Q (256 bytes) -> (status name, P + Q, 128 bytes)."""
    return _eth_evm_ecop("bls12381_g1add", inputs, out_len)


def eth_evm_bls12381_g2add(inputs: bytes, out_len: int = 256):
    """EIP-2537 BLS12_G2ADD through ctt_eth_evm_bls12381_g2add: P, Q (512 bytes) -> (status name, P + Q, 256 bytes)."""
    return _eth_evm_ecop("bls12381_g2add", inputs, out_len)


def eth_evm_bls12381_g1mul(inputs: bytes, out_len: int = 128):
    """EIP-2537 BLS12_G1MUL through ctt_eth_evm_bls12381_g1mul: P and a 32-byte scalar (160 bytes) -> (status name, [s]P, 128
    bytes); P must be in G1."""
    return _eth_evm_ecop("bls12381_g1mul", inputs, out_len)


def eth_evm_bls12381_g2mul(inputs: bytes, out_len: int = 256):
    """EIP-2537 BLS12_G2MUL through ctt_eth_evm_bls12381_g2mul: P and a 32-byte scalar (288 bytes) -> (status name, [s]P, 256
    bytes); P must be in G2."""
    return _eth_evm_ecop("bls12381_g2mul", inputs, out_len)


def _eth_evm_ecop_batch(name, data):
    return _eth_evm_records_batch("ctt_b200_eth_evm_" + name + "_batch", data, *ECOPS[name])


def eth_evm_bn254_g1add_batch(data: bytes):
    """n ECADD calls in one pass (ctt_b200_eth_evm_bn254_g1add_batch): data is n x 128 bytes; returns ([status name] * n, n x 64
    output bytes), a failed record's output zeros."""
    return _eth_evm_ecop_batch("bn254_g1add", data)


def eth_evm_bn254_g1mul_batch(data: bytes):
    """n ECMUL calls in one pass: data is n x 96 bytes; returns ([status name] * n, n x 64 output bytes)."""
    return _eth_evm_ecop_batch("bn254_g1mul", data)


def eth_evm_bls12381_g1add_batch(data: bytes):
    """n BLS12_G1ADD calls in one pass: data is n x 256 bytes; returns ([status name] * n, n x 128 output bytes)."""
    return _eth_evm_ecop_batch("bls12381_g1add", data)


def eth_evm_bls12381_g2add_batch(data: bytes):
    """n BLS12_G2ADD calls in one pass: data is n x 512 bytes; returns ([status name] * n, n x 256 output bytes)."""
    return _eth_evm_ecop_batch("bls12381_g2add", data)


def eth_evm_bls12381_g1mul_batch(data: bytes):
    """n BLS12_G1MUL calls in one pass: data is n x 160 bytes; returns ([status name] * n, n x 128 output bytes)."""
    return _eth_evm_ecop_batch("bls12381_g1mul", data)


def eth_evm_bls12381_g2mul_batch(data: bytes):
    """n BLS12_G2MUL calls in one pass: data is n x 288 bytes; returns ([status name] * n, n x 256 output bytes)."""
    return _eth_evm_ecop_batch("bls12381_g2mul", data)


def eth_evm_ecrecover(inputs: bytes, out_len: int = 32):
    """ECRECOVER (precompile 0x01) through ctt_eth_evm_ecrecover: msg || v || r || s (128 bytes, big-endian) -> (status name, 32
    bytes). Only bytes 12..31 are written, with the address of the recovered key; bytes 0..11 come back as zeros. An unrecoverable
    signature succeeds with the zero key's address 0x3f17f1962b36e491b30a40b2405849e597ba5fb5 (see the header for the rules and
    how they differ from geth)."""
    return _eth_evm_ecop("ecrecover", inputs, out_len)


def eth_evm_ecrecover_batch(data: bytes):
    """n ECRECOVER calls in one pass (ctt_b200_eth_evm_ecrecover_batch): data is n x 128 bytes; returns ([status name] * n, n x 32
    output bytes: 12 zero bytes, then the address; all zeros for a malformed record)."""
    return _eth_evm_records_batch("ctt_b200_eth_evm_ecrecover_batch", data, 128, 32)


ECDSA_STATUS = ("cttEthEcdsa_Success", "cttEthEcdsa_VerificationFailure", "cttEthEcdsa_SecretKeyOutOfRange",
                "cttEthEcdsa_SignatureOutOfRange", "cttEthEcdsa_PublicKeyCoordinateOutOfRange", "cttEthEcdsa_PublicKeyNotOnCurve",
                "cttEthEcdsa_NonceFailure")
ECDSA_NONCE = {"random": 0, "rfc6979": 1}   # the reference's NonceSampler order


def _ecdsa_call(name, *args):
    rc = getattr(_lib.load(), "ctt_b200_eth_ecdsa_" + name)(*args)
    if rc < 0:
        raise ValueError("ctt_b200_eth_ecdsa_%s: invalid call" % name)
    return rc


def _ecdsa_one(name, out_size, *args):
    out = ctypes.create_string_buffer(out_size)
    return ECDSA_STATUS[_ecdsa_call(name, out, *args)], out.raw


def eth_ecdsa_sign(seckey: bytes, msg: bytes, nonce: str = "rfc6979"):
    """Ethereum ECDSA signature of msg (hashed with Keccak-256) under the 32-byte big-endian secret key, through
    ctt_b200_eth_ecdsa_sign: (status name, r || s, 64 bytes, low s). nonce: "rfc6979" (deterministic) or "random"."""
    msg = bytes(msg)
    return _ecdsa_one("sign", 64, bytes(seckey), msg, len(msg), ECDSA_NONCE[nonce])


def eth_ecdsa_verify(pubkey: bytes, msg: bytes, sig: bytes) -> str:
    """ctt_b200_eth_ecdsa_verify: the status of sig (r || s) over msg under the 64-byte key x || y."""
    msg = bytes(msg)
    return ECDSA_STATUS[_ecdsa_call("verify", bytes(pubkey), msg, len(msg), bytes(sig))]


def eth_ecdsa_recover_pubkey(msg: bytes, sig: bytes, even_y: bool):
    """ctt_b200_eth_ecdsa_recover_pubkey: (status name, the 64-byte key; zeros when there is none)."""
    msg = bytes(msg)
    return _ecdsa_one("recover_pubkey", 64, msg, len(msg), bytes(sig), int(bool(even_y)))


def eth_ecdsa_recover_pubkey_from_digest(digest: bytes, sig: bytes, even_y: bool):
    """ctt_b200_eth_ecdsa_recover_pubkey_from_digest: a 32-byte digest (taken mod n) instead of the message."""
    return _ecdsa_one("recover_pubkey_from_digest", 64, bytes(digest), bytes(sig), int(bool(even_y)))


def eth_ecdsa_derive_pubkey(seckey: bytes):
    """ctt_b200_eth_ecdsa_derive_pubkey: (status name, [d]G as x || y)."""
    return _ecdsa_one("derive_pubkey", 64, bytes(seckey))


def _ecdsa_joined(items, size, n):
    items = [bytes(x) for x in items]
    if len(items) != n or any(len(x) != size for x in items):
        raise ValueError("%d items of %d bytes expected" % (n, size))
    return b"".join(items)


def _ecdsa_messages(msgs):
    offsets, data = _offsets([bytes(m) for m in msgs])
    return data, offsets[len(msgs)], offsets


def _ecdsa_batch(name, n, out_size, *args):
    """n items through ctt_b200_eth_ecdsa_<name>_batch: [(status name, out_size output bytes)], or [status name] for out_size 0"""
    if n == 0:
        return []
    st = ctypes.create_string_buffer(n)
    if not out_size:
        _ecdsa_call(name + "_batch", st, *args)
        return [ECDSA_STATUS[b] for b in st.raw]
    out = ctypes.create_string_buffer(out_size * n)
    _ecdsa_call(name + "_batch", out, st, *args)
    return [(ECDSA_STATUS[st.raw[i]], out.raw[out_size * i:out_size * (i + 1)]) for i in range(n)]


def eth_ecdsa_sign_batch(seckeys, msgs, nonce: str = "rfc6979") -> list:
    """n signatures in one pass (ctt_b200_eth_ecdsa_sign_batch): lists of secret keys and messages -> [(status name, r || s)]."""
    n = len(msgs)
    return _ecdsa_batch("sign", n, 64, _ecdsa_joined(seckeys, 32, n), *_ecdsa_messages(msgs), n, ECDSA_NONCE[nonce])


def eth_ecdsa_verify_batch(pubkeys, msgs, sigs) -> list:
    """n verifications in one pass (ctt_b200_eth_ecdsa_verify_batch) -> [status name]."""
    n = len(msgs)
    return _ecdsa_batch("verify", n, 0, _ecdsa_joined(pubkeys, 64, n), _ecdsa_joined(sigs, 64, n), *_ecdsa_messages(msgs), n)


def eth_ecdsa_recover_pubkey_batch(msgs, sigs, even_y) -> list:
    """n recoveries in one pass (ctt_b200_eth_ecdsa_recover_pubkey_batch) -> [(status name, 64-byte key)]."""
    n = len(msgs)
    ev = _ecdsa_joined([b"\1" if e else b"\0" for e in even_y], 1, n)
    return _ecdsa_batch("recover_pubkey", n, 64, _ecdsa_joined(sigs, 64, n), ev, *_ecdsa_messages(msgs), n)


def eth_ecdsa_recover_pubkey_from_digest_batch(digests, sigs, even_y) -> list:
    """n recoveries from 32-byte digests in one pass (ctt_b200_eth_ecdsa_recover_pubkey_from_digest_batch)."""
    n = len(digests)
    ev = _ecdsa_joined([b"\1" if e else b"\0" for e in even_y], 1, n)
    return _ecdsa_batch("recover_pubkey_from_digest", n, 64, _ecdsa_joined(digests, 32, n), _ecdsa_joined(sigs, 64, n), ev, n)


def eth_ecdsa_derive_pubkey_batch(seckeys) -> list:
    """n public keys in one pass (ctt_b200_eth_ecdsa_derive_pubkey_batch) -> [(status name, x || y)]."""
    n = len(seckeys)
    return _ecdsa_batch("derive_pubkey", n, 64, _ecdsa_joined(seckeys, 32, n), n)


def eth_ecdsa_last_timing() -> dict:
    """The calling thread's last ECDSA call: host work before the kernel and the kernel's CUDA-event time (ms)."""
    h, k = ctypes.c_float(0), ctypes.c_float(0)
    _lib.load().ctt_b200_eth_ecdsa_last_timing(ctypes.byref(h), ctypes.byref(k))
    return {"ms_host": h.value, "ms_kernel": k.value}


def eth_evm_sha256(inputs: bytes, out_len: int = 32):
    """SHA256 (precompile 0x02) through ctt_eth_evm_sha256: any message -> (status name, 32-byte digest)."""
    return _eth_evm_ecop("sha256", inputs, out_len)


def eth_evm_ripemd160(inputs: bytes, out_len: int = 32):
    """RIPEMD160 (precompile 0x03) through ctt_eth_evm_ripemd160: any message -> (status name, 12 zero bytes || 20-byte digest)."""
    return _eth_evm_ecop("ripemd160", inputs, out_len)


def eth_evm_modexp_result_size(inputs: bytes):
    """ctt_eth_evm_modexp_result_size: (status name, mL), the output length eth_evm_modexp needs for this input."""
    inputs = bytes(inputs)
    v = ctypes.c_uint64(0)
    st = _lib.load().ctt_eth_evm_modexp_result_size(ctypes.byref(v), inputs, len(inputs))
    return EVM_STATUS[st], v.value


def eth_evm_modexp(inputs: bytes, out_len: int = None):
    """MODEXP (precompile 0x05) through ctt_eth_evm_modexp: bL || eL || mL (32 bytes each) || base || exponent || modulus ->
    (status name, b^e mod M in mL big-endian bytes). out_len defaults to result_size's mL (see the header for the rules)."""
    inputs = bytes(inputs)
    if out_len is None:
        st, out_len = eth_evm_modexp_result_size(inputs)
        if st != "cttEVM_Success":
            return st, b""
    return _eth_evm_ecop("modexp", inputs, out_len)


def _offsets(calls):
    k = len(calls)
    offsets = (ctypes.c_size_t * (k + 1))()
    for i, c in enumerate(calls):
        offsets[i + 1] = offsets[i] + len(c)
    return offsets, b"".join(calls) or b"\0"


def _eth_evm_hash_batch(name, calls) -> list:
    calls = [bytes(c) for c in calls]
    k = len(calls)
    if k == 0:
        return []
    offsets, data = _offsets(calls)
    r = ctypes.create_string_buffer(32 * k)
    st = getattr(_lib.load(), name)(r, data, offsets[k], offsets, k)
    if st != 0:
        raise ValueError(EVM_STATUS[st])
    raw = r.raw
    return [raw[32 * i:32 * i + 32] for i in range(k)]


def eth_evm_sha256_batch(calls) -> list:
    """k SHA256 calls of any lengths in one pass (ctt_b200_eth_evm_sha256_batch): a list of messages -> a list of 32-byte digests."""
    return _eth_evm_hash_batch("ctt_b200_eth_evm_sha256_batch", calls)


def eth_evm_ripemd160_batch(calls) -> list:
    """k RIPEMD160 calls in one pass (ctt_b200_eth_evm_ripemd160_batch): a list of messages -> a list of 32-byte outputs."""
    return _eth_evm_hash_batch("ctt_b200_eth_evm_ripemd160_batch", calls)


def eth_evm_modexp_batch(calls, out_lens=None) -> list:
    """k MODEXP calls of any lengths in one pass (ctt_b200_eth_evm_modexp_batch): a list of inputs -> [(status name, output)].
    Output lengths default to each call's result_size (0 where that fails); a failed call's output is zeros."""
    calls = [bytes(c) for c in calls]
    k = len(calls)
    if k == 0:
        return []
    if out_lens is None:
        out_lens = []
        for c in calls:
            st, n = eth_evm_modexp_result_size(c)
            out_lens.append(n if st == "cttEVM_Success" else 0)
    offsets, data = _offsets(calls)
    r_offsets = (ctypes.c_size_t * (k + 1))()
    for i, n in enumerate(out_lens):
        r_offsets[i + 1] = r_offsets[i] + n
    r = ctypes.create_string_buffer(max(r_offsets[k], 1))
    statuses = ctypes.create_string_buffer(k)
    st = _lib.load().ctt_b200_eth_evm_modexp_batch(r, statuses, r_offsets, data, offsets[k], offsets, k)
    if st != 0:
        raise ValueError(EVM_STATUS[st])
    raw = r.raw
    return [(EVM_STATUS[statuses.raw[i]], raw[r_offsets[i]:r_offsets[i + 1]]) for i in range(k)]


def eth_evm_ecops_last_timing() -> dict:
    """The kernel time (ms, CUDA events, first kernel to last) of the calling thread's last call of the curve addition /
    multiplication, ecrecover, SHA256, RIPEMD160 or MODEXP entries above; 0 when that call did no device work."""
    v = ctypes.c_float(0)
    _lib.load().ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(v))
    return {"ms_kernel": v.value}


class CtSpan(ctypes.Structure):
    """ctt_span: {byte* data; size_t len} (reference include/constantine/protocols/ethereum_bls_signatures.h:64)."""
    _fields_ = [("data", ctypes.c_void_p), ("len", ctypes.c_size_t)]


ETH_BLS_PUBKEY_BYTES, ETH_BLS_SIGNATURE_BYTES = 96, 192   # affine Montgomery structs (ctt_eth_bls_pubkey / ctt_eth_bls_signature)


def eth_bls_deserialize_pubkey(b48: bytes) -> bytes:
    """48-byte compressed public key -> the 96-byte ctt_eth_bls_pubkey struct (curve and subgroup checked). Raises
    ValueError(status) with the reference's ctt_codec_ecc_status when it is not Success (5 = PointAtInfinity included)."""
    if len(b48) != 48:
        raise ValueError("a compressed public key is 48 bytes, got %d" % len(b48))
    out = ctypes.create_string_buffer(ETH_BLS_PUBKEY_BYTES)
    st = _lib.load().ctt_b200_eth_bls_deserialize_pubkey_compressed(out, _buf(bytes(b48)))
    if st != 0:
        raise ValueError(st)
    return out.raw


def eth_bls_deserialize_signature(b96: bytes) -> bytes:
    """96-byte compressed signature -> the 192-byte ctt_eth_bls_signature struct, as eth_bls_deserialize_pubkey."""
    if len(b96) != 96:
        raise ValueError("a compressed signature is 96 bytes, got %d" % len(b96))
    out = ctypes.create_string_buffer(ETH_BLS_SIGNATURE_BYTES)
    st = _lib.load().ctt_b200_eth_bls_deserialize_signature_compressed(out, _buf(bytes(b96)))
    if st != 0:
        raise ValueError(st)
    return out.raw


def _compressed_items(items, size, what):
    """A list of compressed points, or one joined buffer of them, as (bytes, count); a wrong size raises ValueError."""
    if isinstance(items, (bytes, bytearray, memoryview)):
        b = bytes(items)
        if len(b) % size:
            raise ValueError("joined compressed %ss: %d bytes is not a multiple of %d" % (what, len(b), size))
        return b, len(b) // size
    items = [bytes(x) for x in items]
    for x in items:
        if len(x) != size:
            raise ValueError("a compressed %s is %d bytes, got %d" % (what, size, len(x)))
    return b"".join(items), len(items)


def _deserialize_batch(fn, items, in_size, out_size, what):
    src, n = _compressed_items(items, in_size, what)
    if n == 0:
        return [], []
    out = ctypes.create_string_buffer(out_size * n)
    st = ctypes.create_string_buffer(n)
    rc = fn(out, st, _buf(src), n)
    if rc not in (0, 1):
        raise ValueError("%s batch: %d items rejected by the C entry (rc %d)" % (what, n, rc))
    raw = out.raw
    return [raw[out_size * i:out_size * (i + 1)] for i in range(n)], list(st.raw)


def eth_bls_deserialize_pubkeys(b48s):
    """Compressed public keys decoded on the GPU (ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch): b48s is a list of 48-byte
    keys or one joined buffer of them. Returns (structs, statuses): the 96-byte ctt_eth_bls_pubkey of every key (all zeros unless its
    status is 0) and its ctt_codec_ecc_status, as eth_bls_deserialize_pubkey reports it."""
    return _deserialize_batch(_lib.load().ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch, b48s, 48, ETH_BLS_PUBKEY_BYTES,
                              "public key")


def eth_bls_deserialize_signatures(b96s):
    """Compressed signatures decoded on the GPU (ctt_b200_eth_bls_deserialize_signatures_compressed_batch), as
    eth_bls_deserialize_pubkeys: (192-byte ctt_eth_bls_signature structs, statuses)."""
    return _deserialize_batch(_lib.load().ctt_b200_eth_bls_deserialize_signatures_compressed_batch, b96s, 96, ETH_BLS_SIGNATURE_BYTES,
                              "signature")


def eth_bls_registry_from_compressed(pubkeys) -> "CachedBases":
    """A signature-set registry decoded on the GPU from compressed public keys (ctt_b200_eth_bls_registry_from_compressed): a
    CachedBases of bls12_381_g1 holding the rows CachedBases("bls12_381_g1", structs) would hold. The keys never return to the host.
    A key whose status is not 0 (infinity, 5, included) raises ValueError((status, index)) for the lowest such key; no keys raise
    ValueError((-1, None))."""
    src, n = _compressed_items(pubkeys, 48, "public key")
    failed, status = ctypes.c_size_t(0), ctypes.c_int(0)
    h = _lib.load().ctt_b200_eth_bls_registry_from_compressed(_buf(src or b"\0"), n, None, ctypes.byref(failed), ctypes.byref(status))
    if not h:
        raise ValueError((status.value, None if status.value < 0 else failed.value))
    return CachedBases._from_handle("bls12_381_g1", h, n)


def _eth_bls_items(items, size, what):
    for x in items:
        if len(x) != size:
            raise ValueError("every %s struct is %d bytes, got %d" % (what, size, len(x)))
    return b"".join(bytes(x) for x in items)


def _eth_bls_spans(messages):
    keep = [ctypes.create_string_buffer(bytes(m), max(1, len(m))) for m in messages]
    spans = (CtSpan * max(1, len(messages)))()
    for i, (m, b) in enumerate(zip(messages, keep)):
        spans[i].data = ctypes.cast(b, ctypes.c_void_p)
        spans[i].len = len(m)
    return spans, keep


def eth_bls_batch_verify(pubkeys, messages, signatures, secure_random_bytes: bytes) -> bool:
    """ctt_eth_bls_batch_verify over lists of public key structs (96 bytes), messages and signature structs (192 bytes). True on
    Success; False on VerificationFailure, ZeroLengthAggregation (empty lists) or PointAtInfinity. Lists of unequal length or
    items of the wrong size raise ValueError before the call."""
    if not (len(pubkeys) == len(messages) == len(signatures)):
        raise ValueError("pubkeys, messages and signatures differ in length: %d, %d, %d" % (len(pubkeys), len(messages), len(signatures)))
    if len(secure_random_bytes) != 32:
        raise ValueError("secure_random_bytes is 32 bytes, got %d" % len(secure_random_bytes))
    pk = _eth_bls_items(pubkeys, ETH_BLS_PUBKEY_BYTES, "public key")
    sg = _eth_bls_items(signatures, ETH_BLS_SIGNATURE_BYTES, "signature")
    spans, _keep = _eth_bls_spans(messages)
    st = _lib.load().ctt_eth_bls_batch_verify(_buf(pk or b"\0"), spans, _buf(sg or b"\0"), len(pubkeys), _buf(bytes(secure_random_bytes)))
    if st not in (0, 1, 3, 4):
        raise ValueError(st)
    return st == 0


def eth_bls_aggregate_verify(pubkeys, messages, aggregate_sig: bytes) -> bool:
    """ctt_eth_bls_aggregate_verify: the public keys (96-byte structs) each signed its message, and aggregate_sig (a 192-byte struct)
    is the sum of their signatures. Return values and errors as eth_bls_batch_verify."""
    if len(pubkeys) != len(messages):
        raise ValueError("pubkeys and messages differ in length: %d, %d" % (len(pubkeys), len(messages)))
    pk = _eth_bls_items(pubkeys, ETH_BLS_PUBKEY_BYTES, "public key")
    sg = _eth_bls_items([aggregate_sig], ETH_BLS_SIGNATURE_BYTES, "signature")
    spans, _keep = _eth_bls_spans(messages)
    st = _lib.load().ctt_eth_bls_aggregate_verify(_buf(pk or b"\0"), spans, len(pubkeys), _buf(sg))
    if st not in (0, 1, 3, 4):
        raise ValueError(st)
    return st == 0


def _eth_bls_sets(registry, sets):
    """The C arrays of a list of signature sets (indices, message, signature struct) over a CachedBases registry of BLS12-381 G1
    public keys. Wrong sizes or a registry of another curve raise ValueError."""
    if not isinstance(registry, CachedBases) or registry.curve.name != "bls12_381_g1" or not registry._h:
        raise ValueError("the registry is a CachedBases of bls12_381_g1 public keys")
    indices, counts, msgs, sigs = [], [], [], []
    for k, (idx, msg, sig) in enumerate(sets):
        idx = [int(x) for x in idx]
        if any(x < 0 or x >= 1 << 64 for x in idx):
            raise ValueError("set %d: a key index is not a uint64" % k)
        indices += idx
        counts.append(len(idx))
        msgs.append(bytes(msg))
        sigs.append(sig)
    if len(counts) > 0x7fffffff or len(indices) > 0x7fffffff:
        raise ValueError("more than 2^31 - 1 sets or keys")
    sg = _eth_bls_items(sigs, ETH_BLS_SIGNATURE_BYTES, "signature")
    spans, keep = _eth_bls_spans(msgs)
    idx_arr = (ctypes.c_uint64 * max(1, len(indices)))(*indices)
    cnt_arr = (ctypes.c_size_t * max(1, len(counts)))(*counts)
    return idx_arr, cnt_arr, spans, ctypes.create_string_buffer(sg or b"\0", max(1, len(sg))), len(counts), keep


def eth_bls_batch_verify_sets(registry, sets, secure_random_bytes: bytes) -> bool:
    """ctt_b200_eth_bls_batch_verify_sets: every set (indices into the registry, message, 192-byte signature struct) is a
    fast_aggregate_verify, checked together with one blinding scalar per set. registry: CachedBases("bls12_381_g1", pubkey_structs).
    True on Success, False on VerificationFailure. A set that fails its input checks (status 2 index out of range, 3 no keys, 4 an
    infinity signature or key) raises ValueError((status, failed_set)) for the lowest such set; no sets raise ValueError((3, None))."""
    if len(secure_random_bytes) != 32:
        raise ValueError("secure_random_bytes is 32 bytes, got %d" % len(secure_random_bytes))
    idx, cnt, spans, sg, n, _keep = _eth_bls_sets(registry, sets)
    failed = ctypes.c_size_t(ctypes.c_size_t(-1).value)
    st = _lib.load().ctt_b200_eth_bls_batch_verify_sets(registry._h, idx, cnt, spans, sg, n, _buf(bytes(secure_random_bytes)),
                                                         ctypes.byref(failed))
    if st in (0, 1):
        return st == 0
    raise ValueError((st, None if failed.value == ctypes.c_size_t(-1).value else failed.value))


def eth_bls_verify_sets(registry, sets) -> list:
    """ctt_b200_eth_bls_verify_sets: the reference's fast_aggregate_verify status of every set (0 Success, 1 VerificationFailure,
    2 a key index out of range, 3 no keys, 4 an infinity signature or key), no blinding. Arguments as eth_bls_batch_verify_sets;
    no sets give []."""
    idx, cnt, spans, sg, n, _keep = _eth_bls_sets(registry, sets)
    if n == 0:
        return []
    out = ctypes.create_string_buffer(n)
    st = _lib.load().ctt_b200_eth_bls_verify_sets(registry._h, idx, cnt, spans, sg, n, out)
    if st not in (0, 1):
        raise ValueError(st)
    return list(out.raw)


def eth_bls_last_timing() -> dict:
    """Host checks with expand_message_xmd and the blinding chain, device hash to G2, blinding, Miller loops, final exponentiation
    (CUDA events) and the G2 MSM (ms) of the calling thread's last BLS verification."""
    v = [ctypes.c_float(0) for _ in range(6)]
    _lib.load().ctt_b200_eth_bls_last_timing(*[ctypes.byref(x) for x in v])
    return dict(zip(("ms_host", "ms_hash", "ms_blind", "ms_msm", "ms_miller", "ms_final"), (x.value for x in v)))


BLS_SCALAR_STATUS = ("cttCodecScalar_Success", "cttCodecScalar_Zero", "cttCodecScalar_ScalarLargerThanCurveOrder")


def _bls_sign_call(name, *args):
    rc = getattr(_lib.load(), "ctt_b200_eth_bls_" + name)(*args)
    if rc < 0:
        raise ValueError("ctt_b200_eth_bls_%s: invalid call" % name)
    return rc


def _bls_sign_batch(name, n, out_size, *args):
    if n == 0:
        return []
    st = ctypes.create_string_buffer(n)
    out = ctypes.create_string_buffer(out_size * n)
    _bls_sign_call(name + "_batch", out, st, *args)
    sts, raw = st.raw, out.raw
    return [(BLS_SCALAR_STATUS[sts[i]], raw[out_size * i:out_size * (i + 1)]) for i in range(n)]


def eth_bls_sign(seckey: bytes, msg: bytes):
    """Ethereum BLS signature of msg (DST BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_) under the 32-byte big-endian secret key,
    through ctt_b200_eth_bls_sign: (status name, 96-byte compressed signature; zeros unless the status is Success)."""
    msg = bytes(msg)
    out = ctypes.create_string_buffer(96)
    return BLS_SCALAR_STATUS[_bls_sign_call("sign", out, bytes(seckey), msg, len(msg))], out.raw


def eth_bls_derive_pubkey(seckey: bytes):
    """ctt_b200_eth_bls_derive_pubkey: (status name, 48-byte compressed [sk]G1)."""
    out = ctypes.create_string_buffer(48)
    return BLS_SCALAR_STATUS[_bls_sign_call("derive_pubkey", out, bytes(seckey))], out.raw


def eth_bls_sign_batch(seckeys, msgs) -> list:
    """n signatures in one pass (ctt_b200_eth_bls_sign_batch): lists of secret keys and messages -> [(status name, 96 bytes)]."""
    n = len(msgs)
    return _bls_sign_batch("sign", n, 96, _ecdsa_joined(seckeys, 32, n), *_ecdsa_messages(msgs), n)


def eth_bls_derive_pubkey_batch(seckeys) -> list:
    """n public keys in one pass (ctt_b200_eth_bls_derive_pubkey_batch) -> [(status name, 48 bytes)]."""
    n = len(seckeys)
    return _bls_sign_batch("derive_pubkey", n, 48, _ecdsa_joined(seckeys, 32, n), n)


def _serialize_batch(name, items, in_size, out_size, what):
    src, n = _compressed_items(items, in_size, what)
    if n == 0:
        return []
    out = ctypes.create_string_buffer(out_size * n)
    _bls_sign_call(name, out, _buf(src), n)
    raw = out.raw
    return [raw[out_size * i:out_size * (i + 1)] for i in range(n)]


def eth_bls_serialize_pubkeys(pubkeys) -> list:
    """ctt_eth_bls_pubkey structs (96 bytes, a list or one joined buffer) compressed on the GPU
    (ctt_b200_eth_bls_serialize_pubkeys_compressed_batch) -> [48 bytes]."""
    return _serialize_batch("serialize_pubkeys_compressed_batch", pubkeys, ETH_BLS_PUBKEY_BYTES, 48, "public key struct")


def eth_bls_serialize_signatures(sigs) -> list:
    """ctt_eth_bls_signature structs (192 bytes) compressed on the GPU (ctt_b200_eth_bls_serialize_signatures_compressed_batch)
    -> [96 bytes]."""
    return _serialize_batch("serialize_signatures_compressed_batch", sigs, ETH_BLS_SIGNATURE_BYTES, 96, "signature struct")


def eth_bls_serialize_pubkey(pubkey: bytes) -> bytes:
    """ctt_b200_eth_bls_serialize_pubkey_compressed on the host: a 96-byte struct -> 48 bytes."""
    out = ctypes.create_string_buffer(48)
    _bls_sign_call("serialize_pubkey_compressed", out, _buf(_compressed_items([pubkey], ETH_BLS_PUBKEY_BYTES, "public key struct")[0]))
    return out.raw


def eth_bls_serialize_signature(sig: bytes) -> bytes:
    """ctt_b200_eth_bls_serialize_signature_compressed on the host: a 192-byte struct -> 96 bytes."""
    out = ctypes.create_string_buffer(96)
    _bls_sign_call("serialize_signature_compressed", out, _buf(_compressed_items([sig], ETH_BLS_SIGNATURE_BYTES, "signature struct")[0]))
    return out.raw


def eth_bls_signer_last_timing() -> dict:
    """The calling thread's last BLS signing call (ms): host expand_message_xmd, the hash-to-G2 kernel and the multiplication and
    compression kernel (CUDA events)."""
    v = [ctypes.c_float(0) for _ in range(3)]
    _lib.load().ctt_b200_eth_bls_signer_last_timing(*[ctypes.byref(x) for x in v])
    return dict(zip(("ms_host", "ms_hash", "ms_kernel"), (x.value for x in v)))


EIP2333_SEED_STATUS = ("Success", "SeedTooShort")


def eip2334_path(path: str) -> list:
    """An EIP-2334 path string ("m/12381/3600/0/0/0") -> its child indices ([12381, 3600, 0, 0, 0]); "m" alone is []. Each index is
    canonical decimal (no sign, no leading zero, no hardening mark) below 2^32; anything else raises ValueError."""
    parts = path.split("/")
    if parts[0] != "m":
        raise ValueError("an EIP-2334 path starts with m: %r" % path)
    out = []
    for p in parts[1:]:
        if not p or not p.isascii() or not p.isdigit() or (len(p) > 1 and p[0] == "0") or int(p) >= 1 << 32:
            raise ValueError("bad EIP-2334 path component %r in %r" % (p, path))
        out.append(int(p))
    return out


def _eip2333_call(name, *args):
    rc = getattr(_lib.load(), "ctt_b200_eth_eip2333_" + name)(*args)
    if rc < 0:
        raise ValueError("ctt_b200_eth_eip2333_%s: invalid call" % name)
    return rc


def _eip2333_index(i):
    """an index as the C entries take it, a uint32_t: ValueError outside [0, 2^32) rather than ctypes' silent wrap-around"""
    i = operator.index(i)
    if not 0 <= i < 1 << 32:
        raise ValueError("index %d is outside [0, 2^32)" % i)
    return i


def _eip2333_indices(indices, n):
    indices = [_eip2333_index(i) for i in indices]
    if len(indices) != n:
        raise ValueError("%d indices expected" % n)
    return (ctypes.c_uint32 * max(n, 1))(*indices)


def eth_eip2333_derive_master_secret_key(ikm: bytes):
    """EIP-2333 derive_master_SK(IKM) through ctt_b200_eth_eip2333_derive_master_secret_key: (status name of EIP2333_SEED_STATUS,
    32-byte big-endian key; zeros for an IKM shorter than 32 bytes)."""
    ikm = bytes(ikm)
    out = ctypes.create_string_buffer(32)
    return EIP2333_SEED_STATUS[_eip2333_call("derive_master_secret_key", out, ikm, len(ikm))], out.raw


def eth_eip2333_derive_child_secret_key(parent: bytes, index: int):
    """EIP-2333 derive_child_SK(parent, index) through ctt_b200_eth_eip2333_derive_child_secret_key: (the parent's
    BLS_SCALAR_STATUS name, 32-byte key; zeros unless Success)."""
    out = ctypes.create_string_buffer(32)
    return BLS_SCALAR_STATUS[_eip2333_call("derive_child_secret_key", out, _ecdsa_joined([parent], 32, 1), _eip2333_index(index))], out.raw


def eth_eip2333_derive_master_secret_keys_batch(ikms) -> list:
    """n master keys in one pass (ctt_b200_eth_eip2333_derive_master_secret_keys_batch) -> [(status name, 32 bytes)]."""
    ikms = list(ikms)
    n = len(ikms)
    if n == 0:
        return []
    st, out = ctypes.create_string_buffer(n), ctypes.create_string_buffer(32 * n)
    _eip2333_call("derive_master_secret_keys_batch", out, st, *_ecdsa_messages(ikms), n)
    raw = out.raw
    return [(EIP2333_SEED_STATUS[st.raw[i]], raw[32 * i:32 * i + 32]) for i in range(n)]


def eth_eip2333_derive_child_secret_keys_batch(parents, indices) -> list:
    """n child keys in one pass (ctt_b200_eth_eip2333_derive_child_secret_keys_batch): parents (32 bytes each) and their indices
    -> [(status name, 32 bytes)]."""
    parents = list(parents)
    n = len(parents)
    if n == 0:
        return []
    idx = _eip2333_indices(indices, n)
    st, out = ctypes.create_string_buffer(n), ctypes.create_string_buffer(32 * n)
    _eip2333_call("derive_child_secret_keys_batch", out, st, _ecdsa_joined(parents, 32, n), idx, n)
    raw = out.raw
    return [(BLS_SCALAR_STATUS[st.raw[i]], raw[32 * i:32 * i + 32]) for i in range(n)]


def eth_eip2333_derive_path_batch(seeds, seed_of, paths, secret_keys: bool = True, pubkeys: bool = True) -> list:
    """Keys along EIP-2334 paths in one call (ctt_b200_eth_eip2333_derive_path_batch). seeds: the distinct seeds; seed_of[i]: the index
    of item i's seed; paths[i]: its child indices (all of one depth) or a path string for eip2334_path. Common prefixes are derived
    once. -> [(status name of EIP2333_SEED_STATUS, 32-byte key or None, 48-byte compressed public key or None)], with None for an
    output not asked for; with secret_keys=False no secret key leaves the device."""
    seed_of = list(seed_of)
    paths = [eip2334_path(p) if isinstance(p, str) else list(p) for p in paths]
    n = len(seed_of)
    if len(paths) != n:
        raise ValueError("%d paths expected" % n)
    if n == 0:
        return []
    depth = len(paths[0])
    if any(len(p) != depth for p in paths):
        raise ValueError("the paths of one call have one depth")
    data, data_len, offsets = _ecdsa_messages(list(seeds))
    flat = _eip2333_indices([x for p in paths for x in p], n * depth)
    st = ctypes.create_string_buffer(n)
    sk = ctypes.create_string_buffer(32 * n) if secret_keys else None
    pk = ctypes.create_string_buffer(48 * n) if pubkeys else None
    _eip2333_call("derive_path_batch", sk, pk, st, data, data_len, offsets, len(seeds), _eip2333_indices(seed_of, n), flat, depth, n)
    sks, pks = sk.raw if sk else None, pk.raw if pk else None
    return [(EIP2333_SEED_STATUS[st.raw[i]], sks[32 * i:32 * i + 32] if sks else None, pks[48 * i:48 * i + 48] if pks else None)
            for i in range(n)]


def eth_eip2333_last_stats() -> dict:
    """The calling thread's last key-derivation call: ms_host (path planning), ms_kernel (CUDA events), and the master and child
    derivations that ran."""
    f = [ctypes.c_float(0) for _ in range(2)]
    c = [ctypes.c_uint64(0) for _ in range(2)]
    _lib.load().ctt_b200_eth_eip2333_last_stats(*[ctypes.byref(x) for x in f + c])
    return {"ms_host": f[0].value, "ms_kernel": f[1].value, "masters": c[0].value, "children": c[1].value}


class EthKzgContext:
    """EIP-4844 commitment context on the resident SRS, the role of the reference's EthereumKZGContext for
    blob_to_kzg_commitment[_parallel] (reference constantine/ethereum_eip4844_kzg_parallel.nim:125-159)."""

    ScalarLargerThanCurveOrder = 4        # cttEthKzg_ScalarLargerThanCurveOrder

    def __init__(self, srs_lagrange_brp_g1, compressed=True):
        lib = _lib.load()
        buf = _buf(srs_lagrange_brp_g1)
        if compressed:
            st = ctypes.c_int(0)
            self._h = lib.ctt_b200_eth_kzg_context_new_compressed(buf, ctypes.byref(st))
            if not self._h:
                raise ValueError(f"trusted setup point does not decode (cttEthKzg status {st.value})")
        else:
            self._h = lib.ctt_b200_eth_kzg_context_new(buf)
            if not self._h:
                raise ValueError("ctt_b200_eth_kzg_context_new failed")

    def precompute(self, c: int = 0) -> int:
        return _lib.load().ctt_b200_eth_kzg_context_precompute(self._h, c)

    def blob_to_kzg_commitment(self, blob) -> bytes:
        """48-byte compressed commitment; raises ValueError carrying the reference's status code for an invalid blob."""
        dst = ctypes.create_string_buffer(48)
        rc = _lib.load().ctt_b200_eth_kzg_blob_to_kzg_commitment(self._h, dst, _buf(blob))
        if rc != 0:
            raise ValueError(rc)
        return dst.raw

    # EIP-4844 proofs (reference constantine/ethereum_eip4844_kzg_parallel.nim:161-252). Input lengths are fixed at the C boundary,
    # so a wrong length is refused here with a ValueError carrying a message; a status from the library raises ValueError(status).
    BYTES_PER_BLOB = 4096 * 32

    @staticmethod
    def _check_len(name, b, n):
        if len(memoryview(b).cast("B")) != n:
            raise ValueError(f"{name} must be {n} bytes, got {len(memoryview(b).cast('B'))}")

    def compute_kzg_proof(self, blob, z) -> tuple:
        """(48-byte compressed proof, y = p(z) as 32 big-endian bytes) for the blob opened at z (32 big-endian bytes)."""
        self._check_len("blob", blob, self.BYTES_PER_BLOB)
        self._check_len("z", z, 32)
        proof, y = ctypes.create_string_buffer(48), ctypes.create_string_buffer(32)
        rc = _lib.load().ctt_b200_eth_kzg_compute_kzg_proof(self._h, proof, y, _buf(blob), _buf(z))
        if rc != 0:
            raise ValueError(rc)
        return proof.raw, y.raw

    def compute_blob_kzg_proof(self, blob, commitment) -> bytes:
        """48-byte compressed proof of the blob at the Fiat-Shamir challenge of (blob, commitment)."""
        self._check_len("blob", blob, self.BYTES_PER_BLOB)
        self._check_len("commitment", commitment, 48)
        proof = ctypes.create_string_buffer(48)
        rc = _lib.load().ctt_b200_eth_kzg_compute_blob_kzg_proof(self._h, proof, _buf(blob), _buf(commitment))
        if rc != 0:
            raise ValueError(rc)
        return proof.raw

    def _batch(self, blobs, per_item=None, name="commitments"):
        blobs = [bytes(b) for b in blobs]
        for b in blobs:
            self._check_len("blob", b, self.BYTES_PER_BLOB)
        if per_item is not None:
            per_item = [bytes(c) for c in per_item]
            if len(per_item) != len(blobs):
                raise ValueError(f"{len(blobs)} blobs but {len(per_item)} {name}")
            for c in per_item:
                self._check_len(name[:-1], c, 48)
        return blobs, per_item

    def blobs_to_kzg_commitments(self, blobs) -> list:
        """Commitments of several blobs in one pass of the engine. A bad blob raises ValueError(status, index) and nothing is
        returned."""
        blobs, _ = self._batch(blobs)
        n = len(blobs)
        out, failed = ctypes.create_string_buffer(max(1, 48 * n)), ctypes.c_size_t(0)
        rc = _lib.load().ctt_b200_eth_kzg_blobs_to_kzg_commitments(self._h, out, _buf(b"".join(blobs) or b"\0"), n, ctypes.byref(failed))
        if rc != 0:
            raise ValueError(rc, failed.value)
        return [out.raw[48 * j:48 * j + 48] for j in range(n)]

    def compute_blob_kzg_proofs(self, blobs, commitments) -> list:
        """Blob proofs of several (blob, commitment) pairs in one pass of the engine. A bad input raises ValueError(status, index)."""
        blobs, commitments = self._batch(blobs, commitments)
        n = len(blobs)
        out, failed = ctypes.create_string_buffer(max(1, 48 * n)), ctypes.c_size_t(0)
        rc = _lib.load().ctt_b200_eth_kzg_compute_blob_kzg_proofs(self._h, out, _buf(b"".join(blobs) or b"\0"),
                                                                 _buf(b"".join(commitments) or b"\0"), n, ctypes.byref(failed))
        if rc != 0:
            raise ValueError(rc, failed.value)
        return [out.raw[48 * j:48 * j + 48] for j in range(n)]

    @staticmethod
    def last_timing() -> dict:
        """Host checks + challenge and quotient-kernel time (ms) of the calling thread's last proof call."""
        h, q = ctypes.c_float(0), ctypes.c_float(0)
        _lib.load().ctt_b200_eth_kzg_last_timing(ctypes.byref(h), ctypes.byref(q))
        return {"ms_host": h.value, "ms_quotient": q.value}

    # EIP-7594 cells and cell proofs (reference constantine/eth_eip7594_peerdas.nim:161-340). Same conventions as above.
    CELLS_PER_EXT_BLOB = 128
    BYTES_PER_CELL = 2048

    def load_peerdas(self, srs_monomial_compressed):
        """One-time: the 4096 monomial-form setup points (48-byte compressed, file order) -> the FK20 bank, resident on the device.
        Raises ValueError(status) if a point does not decode."""
        self._check_len("srs_monomial_compressed", srs_monomial_compressed, 4096 * 48)
        rc = _lib.load().ctt_b200_eth_kzg_context_load_peerdas(self._h, _buf(srs_monomial_compressed))
        if rc != 0:
            raise ValueError(rc)
        self._peerdas_loaded = True

    def _split(self, cells_raw, proofs_raw, n):
        c, k = self.BYTES_PER_CELL, self.CELLS_PER_EXT_BLOB
        cells = [[cells_raw[(j * k + i) * c:(j * k + i + 1) * c] for i in range(k)] for j in range(n)]
        proofs = [[proofs_raw[(j * k + i) * 48:(j * k + i + 1) * 48] for i in range(k)] for j in range(n)] if proofs_raw else None
        return cells, proofs

    def compute_cells(self, blob) -> list:
        """The 128 cells (2048 bytes each) of the extended blob. Works without load_peerdas."""
        self._check_len("blob", blob, self.BYTES_PER_BLOB)
        cells = ctypes.create_string_buffer(self.CELLS_PER_EXT_BLOB * self.BYTES_PER_CELL)
        rc = _lib.load().ctt_b200_eth_kzg_compute_cells(self._h, cells, _buf(blob))
        if rc != 0:
            raise ValueError(rc)
        return self._split(cells.raw, None, 1)[0][0]

    def compute_cells_and_kzg_proofs(self, blob) -> tuple:
        """(128 cells of 2048 bytes, 128 proofs of 48 bytes); needs load_peerdas (without it: ValueError(1))."""
        self._check_len("blob", blob, self.BYTES_PER_BLOB)
        cells = ctypes.create_string_buffer(self.CELLS_PER_EXT_BLOB * self.BYTES_PER_CELL)
        proofs = ctypes.create_string_buffer(self.CELLS_PER_EXT_BLOB * 48)
        rc = _lib.load().ctt_b200_eth_kzg_compute_cells_and_kzg_proofs(self._h, cells, proofs, _buf(blob))
        if rc != 0:
            raise ValueError(rc)
        c, p = self._split(cells.raw, proofs.raw, 1)
        return c[0], p[0]

    def compute_cells_and_kzg_proofs_batch(self, blobs) -> list:
        """[(cells, proofs)] of several blobs in one device pass. A bad blob raises ValueError(status, index) and nothing is returned."""
        blobs, _ = self._batch(blobs)
        n = len(blobs)
        cells = ctypes.create_string_buffer(max(1, n * self.CELLS_PER_EXT_BLOB * self.BYTES_PER_CELL))
        proofs = ctypes.create_string_buffer(max(1, n * self.CELLS_PER_EXT_BLOB * 48))
        failed = ctypes.c_size_t(0)
        rc = _lib.load().ctt_b200_eth_kzg_compute_cells_and_kzg_proofs_batch(self._h, cells, proofs, _buf(b"".join(blobs) or b"\0"), n,
                                                                            ctypes.byref(failed))
        if rc != 0:
            raise ValueError(rc, failed.value)
        c, p = self._split(cells.raw, proofs.raw, n)
        return list(zip(c, p))

    def _recovery_inputs(self, items):
        """[(cell_indices, cells)] -> (uint64 index array, concatenated cells, size_t count array). A cell that is not 2048 bytes, or
        unequal numbers of indices and cells, raise ValueError(str); counts and index values are left to the library's checks."""
        idx, cells, counts = [], [], []
        for j, (cell_indices, blob_cells) in enumerate(items):
            cell_indices, blob_cells = [int(i) for i in cell_indices], [bytes(c) for c in blob_cells]
            if len(cell_indices) != len(blob_cells):
                raise ValueError(f"blob {j}: {len(cell_indices)} cell indices but {len(blob_cells)} cells")
            for c in blob_cells:
                self._check_len("cell", c, self.BYTES_PER_CELL)
            idx += cell_indices
            cells += blob_cells
            counts.append(len(blob_cells))
        return (ctypes.c_uint64 * max(1, len(idx)))(*idx), _buf(b"".join(cells) or b"\0"), (ctypes.c_size_t * max(1, len(counts)))(*counts)

    def recover_cells_and_kzg_proofs(self, cell_indices, cells) -> tuple:
        """(128 cells, 128 proofs) of the extended blob from at least 64 of its cells and their ascending indices; needs load_peerdas.
        A status from the library raises ValueError(status)."""
        idx, cb, counts = self._recovery_inputs([(cell_indices, cells)])
        out_cells = ctypes.create_string_buffer(self.CELLS_PER_EXT_BLOB * self.BYTES_PER_CELL)
        out_proofs = ctypes.create_string_buffer(self.CELLS_PER_EXT_BLOB * 48)
        rc = _lib.load().ctt_b200_eth_kzg_recover_cells_and_kzg_proofs(self._h, out_cells, out_proofs, idx, cb, counts[0])
        if rc != 0:
            raise ValueError(rc)
        c, p = self._split(out_cells.raw, out_proofs.raw, 1)
        return c[0], p[0]

    def recover_cells_and_kzg_proofs_batch(self, items) -> list:
        """[(cells, proofs)] for several [(cell_indices, cells)] in one device pass. A bad input raises ValueError(status, index) and
        nothing is returned."""
        items = list(items)
        n = len(items)
        idx, cb, counts = self._recovery_inputs(items)
        out_cells = ctypes.create_string_buffer(max(1, n * self.CELLS_PER_EXT_BLOB * self.BYTES_PER_CELL))
        out_proofs = ctypes.create_string_buffer(max(1, n * self.CELLS_PER_EXT_BLOB * 48))
        failed = ctypes.c_size_t(0)
        rc = _lib.load().ctt_b200_eth_kzg_recover_cells_and_kzg_proofs_batch(self._h, out_cells, out_proofs, idx, cb, counts, n,
                                                                            ctypes.byref(failed))
        if rc != 0:
            raise ValueError(rc, failed.value)
        c, p = self._split(out_cells.raw, out_proofs.raw, n)
        return list(zip(c, p))

    # EIP-7594 batch verification (reference constantine/eth_eip7594_peerdas.nim:509-619)
    def load_g2_setup(self, srs_monomial_g2_compressed):
        """One-time: the 65 monomial G2 points of the trusted setup (96-byte compressed, file order), decoded and checked.
        Raises ValueError(status) at the first bad point."""
        self._check_len("srs_monomial_g2_compressed", srs_monomial_g2_compressed, 65 * 96)
        rc = _lib.load().ctt_b200_eth_kzg_context_load_g2_setup(self._h, _buf(srs_monomial_g2_compressed))
        if rc != 0:
            raise ValueError(rc)
        self._g2_loaded = True

    def verify_cell_kzg_proof_batch(self, commitments, cell_indices, cells, proofs, secure_random_bytes=bytes(32)) -> bool:
        """True when every cell k belongs, at column cell_indices[k], to the blob committed to by commitments[k] (proof proofs[k]);
        False when the batch does not verify. Needs load_peerdas and load_g2_setup (else RuntimeError, so False always means "does
        not verify"). Lists of unequal length or items of the wrong size raise ValueError(str); a status from the library (2, 4-8)
        raises ValueError(status). secure_random_bytes: 32 bytes; when they reduce to zero the Fiat-Shamir challenge is used."""
        if not (getattr(self, "_peerdas_loaded", False) and getattr(self, "_g2_loaded", False)):
            raise RuntimeError("verify_cell_kzg_proof_batch needs load_peerdas and load_g2_setup")
        commitments, cells, proofs = [bytes(c) for c in commitments], [bytes(c) for c in cells], [bytes(p) for p in proofs]
        cell_indices = [int(i) for i in cell_indices]
        n = len(cells)
        if not len(commitments) == len(cell_indices) == n == len(proofs):
            raise ValueError(f"{len(commitments)} commitments, {len(cell_indices)} cell indices, {n} cells and {len(proofs)} proofs")
        for c in commitments:
            self._check_len("commitment", c, 48)
        for p in proofs:
            self._check_len("proof", p, 48)
        for c in cells:
            self._check_len("cell", c, self.BYTES_PER_CELL)
        self._check_len("secure_random_bytes", secure_random_bytes, 32)
        idx = (ctypes.c_uint64 * max(1, n))(*cell_indices)
        rc = _lib.load().ctt_b200_eth_kzg_verify_cell_kzg_proof_batch(self._h, _buf(b"".join(commitments) or b"\0"), idx,
                                                                      _buf(b"".join(cells) or b"\0"), _buf(b"".join(proofs) or b"\0"),
                                                                      n, _buf(bytes(secure_random_bytes)))
        if rc not in (0, 1):
            raise ValueError(rc)
        return rc == 0

    # EIP-4844 verification (reference constantine/ethereum_eip4844_kzg.nim:380-570). Same conventions as verify_cell_kzg_proof_batch;
    # these need load_g2_setup only.
    def _need_g2(self, name):
        if not getattr(self, "_g2_loaded", False):
            raise RuntimeError(f"{name} needs load_g2_setup")

    def _verify_status(self, rc) -> bool:
        if rc not in (0, 1):
            raise ValueError(rc)
        return rc == 0

    def verify_kzg_proof(self, commitment, z, y, proof) -> bool:
        """True when proof opens the commitment at z (32 big-endian bytes) to y (32 big-endian bytes); False when it does not."""
        self._need_g2("verify_kzg_proof")
        for name, b, n in (("commitment", commitment, 48), ("z", z, 32), ("y", y, 32), ("proof", proof, 48)):
            self._check_len(name, b, n)
        return self._verify_status(_lib.load().ctt_b200_eth_kzg_verify_kzg_proof(self._h, _buf(bytes(commitment)), _buf(bytes(z)),
                                                                                  _buf(bytes(y)), _buf(bytes(proof))))

    def verify_blob_kzg_proof(self, blob, commitment, proof) -> bool:
        """True when proof opens the commitment at the Fiat-Shamir challenge of (blob, commitment) to the blob's value there."""
        self._need_g2("verify_blob_kzg_proof")
        self._check_len("blob", blob, self.BYTES_PER_BLOB)
        self._check_len("commitment", commitment, 48)
        self._check_len("proof", proof, 48)
        return self._verify_status(_lib.load().ctt_b200_eth_kzg_verify_blob_kzg_proof(self._h, _buf(bytes(blob)), _buf(bytes(commitment)),
                                                                                      _buf(bytes(proof))))

    def verify_blob_kzg_proof_batch(self, blobs, commitments, proofs, secure_random_bytes=bytes(32)) -> bool:
        """True when every (blob, commitment, proof) verifies, checked as one random linear combination in one device pass.
        secure_random_bytes: 32 bytes; when they reduce to zero, r is derived from the opening challenges."""
        self._need_g2("verify_blob_kzg_proof_batch")
        blobs, commitments, proofs = [bytes(b) for b in blobs], [bytes(c) for c in commitments], [bytes(p) for p in proofs]
        n = len(blobs)
        if not len(commitments) == n == len(proofs):
            raise ValueError(f"{n} blobs, {len(commitments)} commitments and {len(proofs)} proofs")
        for b in blobs:
            self._check_len("blob", b, self.BYTES_PER_BLOB)
        for c in commitments:
            self._check_len("commitment", c, 48)
        for p in proofs:
            self._check_len("proof", p, 48)
        self._check_len("secure_random_bytes", secure_random_bytes, 32)
        rc = _lib.load().ctt_b200_eth_kzg_verify_blob_kzg_proof_batch(self._h, _buf(b"".join(blobs) or b"\0"),
                                                                      _buf(b"".join(commitments) or b"\0"),
                                                                      _buf(b"".join(proofs) or b"\0"), n, _buf(bytes(secure_random_bytes)))
        return self._verify_status(rc)

    def verify_kzg_proofs(self, commitments, zs, ys, proofs) -> list:
        """n independent verify_kzg_proof checks in one device pass (ctt_b200_eth_kzg_verify_kzg_proofs): the list of the n statuses,
        each what verify_kzg_proof's C entry returns for that index (0 true, 1 false, 4-8 an input that does not decode). Not a
        random linear combination: every index has its own pairing check."""
        self._need_g2("verify_kzg_proofs")
        cols = [[bytes(x) for x in col] for col in (commitments, zs, ys, proofs)]
        n = len(cols[0])
        if any(len(col) != n for col in cols):
            raise ValueError("commitments, zs, ys and proofs differ in length: %s" % [len(col) for col in cols])
        for name, col, size in zip(("commitment", "z", "y", "proof"), cols, (48, 32, 32, 48)):
            for x in col:
                self._check_len(name, x, size)
        statuses = ctypes.create_string_buffer(max(n, 1))
        rc = _lib.load().ctt_b200_eth_kzg_verify_kzg_proofs(self._h, statuses, *[_buf(b"".join(col) or b"\0") for col in cols], n)
        if rc != 0:
            raise ValueError(rc)
        return list(statuses.raw[:n])

    # The EIP-4844 POINT_EVALUATION precompile (0x0a; reference constantine/ethereum_evm_precompiles.nim:1245-1297) on this context:
    # versioned_hash(32) | z(32) | y(32) | commitment(48) | proof(48) -> FIELD_ELEMENTS_PER_BLOB || r, 32 big-endian bytes each.
    def eth_evm_kzg_point_evaluation(self, inputs, out_len: int = 64):
        """One call through ctt_b200_eth_evm_kzg_point_evaluation: (status name, out_len bytes); the output is written only on
        success (zeros otherwise)."""
        self._need_g2("eth_evm_kzg_point_evaluation")
        inputs = bytes(inputs)
        r = ctypes.create_string_buffer(max(out_len, 1))
        st = _lib.load().ctt_b200_eth_evm_kzg_point_evaluation(self._h, r, out_len, inputs or b"\0", len(inputs))
        return EVM_STATUS[st], r.raw[:out_len]

    def eth_evm_kzg_point_evaluation_batch(self, data):
        """n calls in one pass (ctt_b200_eth_evm_kzg_point_evaluation_batch): data is n x 192 bytes; returns ([status name] * n, n x 64
        output bytes), a failed call's output zeros."""
        self._need_g2("eth_evm_kzg_point_evaluation_batch")
        data = bytes(data)
        if len(data) % 192:
            raise ValueError("inputs must be a multiple of 192 bytes")
        n = len(data) // 192
        r = ctypes.create_string_buffer(max(64 * n, 1))
        statuses = ctypes.create_string_buffer(max(n, 1))
        st = _lib.load().ctt_b200_eth_evm_kzg_point_evaluation_batch(self._h, r, statuses, data or b"\0", n)
        if st != 0:
            raise ValueError(EVM_STATUS[st])
        return [EVM_STATUS[b] for b in statuses.raw[:n]], r.raw[:64 * n]

    @staticmethod
    def last_point_eval_timing() -> dict:
        """Host packing and statuses, the record kernel, the Miller loops and the products with final exponentiations (ms, CUDA
        events) of the calling thread's last verify_kzg_proofs or point-evaluation call."""
        v = [ctypes.c_float(0) for _ in range(4)]
        _lib.load().ctt_b200_eth_kzg_last_point_eval_timing(*[ctypes.byref(x) for x in v])
        return dict(zip(("ms_host", "ms_records", "ms_miller", "ms_final"), (x.value for x in v)))

    @staticmethod
    def last_verify_timing() -> dict:
        """Host checks + challenges, device decode, scalar kernels, bank MSM (CUDA events) and host pairing time (ms) of the calling
        thread's last verification of either family (cells or blobs)."""
        v = [ctypes.c_float(0) for _ in range(5)]
        _lib.load().ctt_b200_eth_kzg_last_verify_timing(*[ctypes.byref(x) for x in v])
        return dict(zip(("ms_host", "ms_decode", "ms_fr", "ms_msm", "ms_pairing"), (x.value for x in v)))

    @staticmethod
    def last_das_timing() -> dict:
        """Host checks + serialisation, Fr kernels, bank MSM and EC FFT time (ms) of the calling thread's last cells / proofs /
        recovery call."""
        v = [ctypes.c_float(0) for _ in range(4)]
        _lib.load().ctt_b200_eth_kzg_last_das_timing(*[ctypes.byref(x) for x in v])
        return dict(zip(("ms_host", "ms_fr", "ms_msm", "ms_ecfft"), (x.value for x in v)))

    def delete(self):
        if self._h:
            _lib.load().ctt_b200_eth_kzg_context_delete(self._h)
            self._h = None
