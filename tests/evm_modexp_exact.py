"""Exact models of the SHA256, RIPEMD160 and MODEXP precompiles (reference constantine/ethereum_evm_precompiles.nim:59-253).

- `transcribed(inputs, r_len)`: the reference entry and `powMod_vartime` (math_arbitrary_precision/arithmetic/bigints_views.nim
  :114-222, limbs_mod2k.nim:80-230) branch for branch on Python integers: the small no-reduction path, the odd modulus
  (a Montgomery fixed-window exponentiation with 64-bit words), the power of two with its Euler and even-base shortcuts, and the
  Koc CRT recombination with a Newton inverse mod 2^k.
- `closed(inputs, r_len)`: the rule the library implements, steps 1-7 of the header with Python's pow.
- `ripemd160(msg)`: pure-Python RIPEMD-160 (hashlib may lack OpenSSL's legacy provider).
Both MODEXP models return (status name, output bytes or None); None means the entry does not write r.
"""
import random

WORD = 64
U64 = (1 << 64) - 1


# ---- MODEXP ------------------------------------------------------------------------------------------------------------------
def lengths(inputs):
    padded = bytes(inputs[:96]) + bytes(max(0, 96 - len(inputs)))
    return [int.from_bytes(padded[32 * j:32 * j + 32], "big") for j in range(3)]


def result_size(inputs):
    mL = lengths(inputs)[2]
    if mL > U64:
        return "cttEVM_InvalidInputSize", None
    return "cttEVM_Success", mL


def _operands(inputs, bL, eL, mL):
    """base, exponent bytes, modulus (zero-padded on the right); the caller has checked 96 + bL + eL < len(inputs)"""
    b = int.from_bytes(inputs[96:96 + bL], "big")
    e = bytes(inputs[96 + bL:96 + bL + eL])
    m_bytes = bytes(inputs[96 + bL + eL:96 + bL + eL + mL])
    m_bytes += bytes(mL - len(m_bytes))
    return b, e, int.from_bytes(m_bytes, "big")


def closed(inputs, r_len):
    bL, eL, mL = lengths(inputs)
    if max(bL, eL, mL) > U64:
        return "cttEVM_InvalidInputSize", None
    if r_len != mL:
        return "cttEVM_InvalidOutputSize", None
    if 96 + bL + eL >= len(inputs) or mL == 0:
        return "cttEVM_Success", bytes(mL)
    if eL == 0:
        return "cttEVM_Success", (1).to_bytes(mL, "big")
    if bL == 0:
        return "cttEVM_Success", bytes(mL)
    b, e, m = _operands(inputs, bL, eL, mL)
    if m < 2:
        return "cttEVM_Success", bytes(mL)
    return "cttEVM_Success", pow(b, int.from_bytes(e, "big"), m).to_bytes(mL, "big")


def _bits(x):
    return x.bit_length()


def _ctz(x):
    return (x & -x).bit_length() - 1


def _pow_odd(a, e_bytes, M, window=4):
    """powOddMod_vartime: eBits = 1 reduces; otherwise Montgomery form with R = 2^(64 L), a fixed window over the exponent bits"""
    e = int.from_bytes(e_bytes, "big")
    if _bits(e) == 1:
        return a % M
    L = (_bits(M) + WORD - 1) // WORD
    R = 1 << (WORD * L)
    m0ninv = (-pow(M, -1, 1 << WORD)) % (1 << WORD)

    def redc(t):                      # word-serial Montgomery reduction, t < M R
        for _ in range(L):
            m = ((t & U64) * m0ninv) & U64
            t = (t + m * M) >> WORD
        return t - M if t >= M else t

    a_mont = (a * R) % M
    one = R % M
    table = [one]
    for _ in range((1 << window) - 1):
        table.append(redc(table[-1] * a_mont))
    acc = one
    nbits = _bits(e)
    top = (nbits + window - 1) // window * window
    for i in range(top - window, -1, -window):
        for _ in range(window):
            acc = redc(acc * acc)
        acc = redc(acc * table[(e >> i) & ((1 << window) - 1)])
    return redc(acc)


def _pow_mod2k(a, e_bytes, k):
    """powMod2k_vartime, LSB-first with its early exits"""
    mask = (1 << k) - 1
    e = int.from_bytes(e_bytes, "big")
    msb = _bits(e) - 1
    if msb == -1:
        return 1 & mask if k else 0
    if msb == 0:
        return a & mask
    if a % 2 == 0:
        if _ctz(a) + msb >= k:
            return 0
    bits_left = msb + 1
    if a % 2 == 1 and k - 1 < bits_left:
        bits_left = k - 1
    r, s = 1, a & mask
    for byte in reversed(e_bytes):
        for i in range(8):
            if (byte >> i) & 1:
                r = (r * s) & mask
            s = (s * s) & mask
            bits_left -= 1
            if bits_left == 0:
                return r
    return r


def _inv_mod2k(a, k):
    """invMod2k_vartime: a word inverse, then Newton x(2 - a x), doubling the correct words"""
    words = max(1, (k + WORD - 1) // WORD)
    x = pow(a & U64, -1, 1 << WORD)
    correct = 1
    while correct * WORD < k:
        w = min(words, 2 * correct)
        mod = 1 << (w * WORD)
        t = (x * a) % mod
        u = (2 - t) % mod
        x = (x * u) % mod
        correct = w
    return x & ((1 << k) - 1)


def pow_mod_vartime(a, e_bytes, M):
    m_bits = _bits(M)
    if m_bits < 2:
        return 0
    e = int.from_bytes(e_bytes, "big")
    e_bits = _bits(e)
    if e_bits == 0:
        return 1
    a_bits = _bits(a)
    if a_bits < 2:
        return a
    if e_bits < WORD and (a_bits >> (WORD - e_bits)) == 0 and (a_bits << e_bits) < m_bits:
        return a ** e
    if M % 2 == 1:
        return _pow_odd(a, e_bytes, M)
    ctz = _ctz(M)
    if m_bits - ctz == 1:
        return _pow_mod2k(a, e_bytes, ctz)
    q = M >> ctz
    a1 = _pow_odd(a, e_bytes, q)
    a2 = _pow_mod2k(a, e_bytes, ctz)
    q_inv = _inv_mod2k(q, ctz)
    y = ((a2 - a1) % (1 << ctz)) * q_inv % (1 << ctz)
    return a1 + q * y


def transcribed(inputs, r_len):
    bL, eL, mL = lengths(inputs)
    if bL > U64 or eL > U64 or mL > U64:
        return "cttEVM_InvalidInputSize", None
    if r_len != mL:
        return "cttEVM_InvalidOutputSize", None
    if 96 + bL + eL >= len(inputs):
        return "cttEVM_Success", bytes(mL)
    if mL == 0:
        return "cttEVM_Success", b""
    if eL == 0:
        return "cttEVM_Success", bytes(mL - 1) + b"\x01"
    if bL == 0:
        return "cttEVM_Success", bytes(mL)
    b, e, m = _operands(inputs, bL, eL, mL)
    return "cttEVM_Success", pow_mod_vartime(b, e, m).to_bytes(mL, "big")


def encode(b, e, m, bL=None, eL=None, mL=None, trunc=None):
    """an input: lengths default to the minimal byte lengths of b, e, m (0 for 0); trunc cuts the input to that many bytes"""
    def nb(x):
        return (x.bit_length() + 7) // 8
    bL = nb(b) if bL is None else bL
    eL = nb(e) if eL is None else eL
    mL = nb(m) if mL is None else mL
    raw = (bL.to_bytes(32, "big") + eL.to_bytes(32, "big") + mL.to_bytes(32, "big") + b.to_bytes(bL, "big") +
           e.to_bytes(eL, "big") + m.to_bytes(mL, "big"))
    return raw if trunc is None else raw[:trunc]


def class_edges():
    """every device class at both edges (32 L and 32 L + 1 bits) and the host path (above 8192 bits)"""
    return [32 * L for L in (8, 16, 32, 64, 128, 256)] + [32 * L + 1 for L in (8, 16, 32, 64, 128)] + [8193, 9000]


def designed_moduli(bits, rnd):
    out = {"2^b-1": (1 << bits) - 1, "2^b+1": (1 << bits) + 1, "3": 3, "2": 2, "2^k": 1 << (bits - 1),
           "odd": rnd.getrandbits(bits) | (1 << (bits - 1)) | 1}
    for k in (1, 31, 32, 33, 255, 4096):
        if k < bits - 1:
            q = rnd.getrandbits(bits - k) | (1 << (bits - k - 1)) | 1
            out["2^%d q" % k] = q << k
    return out


def random_call(rnd, bits=None):
    bits = bits or rnd.choice((8, 64, 255, 256, 257, 511, 512, 513, 1024, 1025, 2048, 4096, 8192, 8193))
    kind = rnd.randrange(4)
    if kind == 0:
        m = rnd.getrandbits(bits) | (1 << (bits - 1)) | 1
    elif kind == 1:
        m = 1 << (bits - 1)
    else:
        k = rnd.randrange(1, max(2, bits - 1))
        m = (rnd.getrandbits(max(1, bits - k)) | 1) << k
        m |= 1 << (bits - 1)
    b = rnd.getrandbits(rnd.choice((8, 256, bits, bits + 64, 3000)))
    e = rnd.choice((1, 2, 3, 0x10001, rnd.getrandbits(rnd.choice((16, 64, 256)))))
    return encode(b, e, m, bL=(b.bit_length() + 7) // 8 + rnd.choice((0, 0, 2)), eL=(e.bit_length() + 7) // 8 + rnd.choice((0, 1)))


# ---- RIPEMD-160 ------------------------------------------------------------------------------------------------------------------
_RL = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 7, 4, 13, 1, 10, 6, 15, 3, 12, 0, 9, 5, 2, 14, 11, 8, 3, 10, 14, 4, 9,
       15, 8, 1, 2, 7, 0, 6, 13, 11, 5, 12, 1, 9, 11, 10, 0, 8, 12, 4, 13, 3, 7, 15, 14, 5, 6, 2, 4, 0, 5, 9, 7, 12, 2, 10, 14, 1,
       3, 8, 11, 6, 15, 13]
_RR = [5, 14, 7, 0, 9, 2, 11, 4, 13, 6, 15, 8, 1, 10, 3, 12, 6, 11, 3, 7, 0, 13, 5, 10, 14, 15, 8, 12, 4, 9, 1, 2, 15, 5, 1, 3, 7,
       14, 6, 9, 11, 8, 12, 2, 10, 0, 4, 13, 8, 6, 4, 1, 3, 11, 15, 0, 5, 12, 2, 13, 9, 7, 10, 14, 12, 15, 10, 4, 1, 5, 8, 7, 6, 2,
       13, 14, 0, 3, 9, 11]
_SL = [11, 14, 15, 12, 5, 8, 7, 9, 11, 13, 14, 15, 6, 7, 9, 8, 7, 6, 8, 13, 11, 9, 7, 15, 7, 12, 15, 9, 11, 7, 13, 12, 11, 13, 6, 7,
       14, 9, 13, 15, 14, 8, 13, 6, 5, 12, 7, 5, 11, 12, 14, 15, 14, 15, 9, 8, 9, 14, 5, 6, 8, 6, 5, 12, 9, 15, 5, 11, 6, 8, 13, 12,
       5, 12, 13, 14, 11, 8, 5, 6]
_SR = [8, 9, 9, 11, 13, 15, 15, 5, 7, 7, 8, 11, 14, 14, 12, 6, 9, 13, 15, 7, 12, 8, 9, 11, 7, 7, 12, 7, 6, 15, 13, 11, 9, 7, 15, 11,
       8, 6, 6, 14, 12, 13, 5, 14, 13, 13, 7, 5, 15, 5, 8, 11, 14, 14, 6, 14, 6, 9, 12, 9, 12, 5, 15, 8, 8, 5, 12, 9, 12, 5, 14, 6,
       8, 13, 6, 5, 15, 13, 11, 11]
_KL = [0x00000000, 0x5A827999, 0x6ED9EBA1, 0x8F1BBCDC, 0xA953FD4E]
_KR = [0x50A28BE6, 0x5C4DD124, 0x6D703EF3, 0x7A6D76E9, 0x00000000]
M32 = 0xFFFFFFFF


def _rol(x, n):
    return ((x << n) | (x >> (32 - n))) & M32


def _f(r, x, y, z):
    if r == 0:
        return x ^ y ^ z
    if r == 1:
        return (x & y) | (~x & z & M32)
    if r == 2:
        return (x | (~y & M32)) ^ z
    if r == 3:
        return (x & z) | (y & ~z & M32)
    return x ^ (y | (~z & M32))


def ripemd160(msg):
    msg = bytes(msg)
    h = [0x67452301, 0xEFCDAB89, 0x98BADCFE, 0x10325476, 0xC3D2E1F0]
    data = msg + b"\x80" + bytes((55 - len(msg)) % 64) + (8 * len(msg)).to_bytes(8, "little")
    for off in range(0, len(data), 64):
        x = [int.from_bytes(data[off + 4 * i:off + 4 * i + 4], "little") for i in range(16)]
        al, bl, cl, dl, el = h
        ar, br, cr, dr, er = h
        for j in range(80):
            r = j // 16
            t = (_rol((al + _f(r, bl, cl, dl) + x[_RL[j]] + _KL[r]) & M32, _SL[j]) + el) & M32
            al, el, dl, cl, bl = el, dl, _rol(cl, 10), bl, t
            t = (_rol((ar + _f(4 - r, br, cr, dr) + x[_RR[j]] + _KR[r]) & M32, _SR[j]) + er) & M32
            ar, er, dr, cr, br = er, dr, _rol(cr, 10), br, t
        t = (h[1] + cl + dr) & M32
        h[1] = (h[2] + dl + er) & M32
        h[2] = (h[3] + el + ar) & M32
        h[3] = (h[4] + al + br) & M32
        h[4] = (h[0] + bl + cr) & M32
        h[0] = t
    return b"".join(w.to_bytes(4, "little") for w in h)


def hash_lengths():
    """message lengths of the hash fixture: 0..300, every block boundary up to 1024 and a few long ones"""
    ls = set(range(301))
    for n in range(64, 1025, 64):
        ls.update((n - 9, n - 8, n - 1, n, n + 1))
    ls.update((4095, 4096, 65537, 1 << 20))
    return sorted(ls)


def hash_message(n, seed=2026):
    return random.Random(seed * 1000003 + n).randbytes(n)
