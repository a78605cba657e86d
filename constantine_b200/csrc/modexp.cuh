// MODEXP (EIP-198) arithmetic on the device: b^e mod M for a modulus supplied at run time, odd or even, up to 8192 bits
// (evm_modexp.cu holds the entries, the host pass and the > 8192-bit host path). DESIGN §4u.
//
// A call of class L (limbs of 32 bits, L in {8, 16, 32, 64, 128, 256}, the smallest with 32 L >= bits(M)) runs on a group of
// TPI lanes, each owning LL = L / TPI consecutive limbs: TPI = 1 (one thread per call, LL = L) for L <= 16, TPI = L / 8 (LL = 8)
// above. Every group operation below degenerates to plain code at TPI = 1.
//
// M = q 2^k with q odd. a1 = b^e mod q in Montgomery form with R = 2^(32 L); a2 = b^e mod 2^k with truncated products; both
// parts are recombined by CRT (Koc 1994) as a1 + q ((a2 - a1) q^-1 mod 2^k). q may fill all 32 L bits (no spare bit), so the
// Montgomery accumulator keeps a carry word above each lane's limbs and the result before its conditional subtraction is < 2q.
//
// Montgomery product (CIOS, lane-distributed): for each limb b_j (broadcast from its owner lane), every lane adds a b_j and m q
// to its limbs, m = t_0 m0' computed by lane 0 and broadcast; the accumulator then shifts right by one limb, the lowest limb of
// each lane moving to the lane below. Each lane's carry word (at its limb LL) joins its limb LL - 1 on that shift, so carries
// never cross lanes inside the loop; they are resolved once at the end, by a ballot of generate / propagate bits.
// Not constant time: every input of a precompile is public.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define MX_HD __host__ __device__ __forceinline__
#else
#define MX_HD inline
#endif

namespace b200 {
namespace modexp {

constexpr int WIN = 4;                     // fixed window bits of the odd-part exponentiation
constexpr int TAB = (1 << WIN) - 1;        // table entries b^1 .. b^15 (Montgomery form)
constexpr int MAX_BITS = 8192;             // largest device modulus (EIP-7823's bound); above, the host path

// one device call: byte ranges in the uploaded input buffer (big-endian integers). The base and the exponent are fully present
// and start at their first non-zero byte; the modulus is m_len bytes starting at its first non-zero byte, of which the first
// m_present are in the buffer and the rest are zeros (the input's right padding).
struct Desc {
  uint64_t b_off, b_len, e_off, e_len, m_off, m_len, m_present;
  uint64_t e_bits;    // significant bits of the exponent, >= 1
  uint64_t out_off;   // 4 L bytes of big-endian result in the output buffer
  uint64_t m_bits;    // significant bits of M, >= 2 (at most 32 L on the device)
  uint64_t k;         // trailing zeros of M
};

MX_HD uint8_t ld_byte(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}

// word `gw` (32 bits, little-endian word order) of X >> shift, X the big-endian integer of `len` bytes at src whose first
// `present` bytes are in memory and the rest zero
MX_HD uint32_t load_word(const uint8_t* src, uint64_t len, uint64_t present, uint64_t shift, uint64_t gw) {
  const uint64_t p = shift + 32 * gw;   // lowest bit of the word
  const uint64_t b0 = p >> 3;
  uint64_t v = 0;
  for (int j = 0; j < 5; j++) {
    const uint64_t le = b0 + j;         // byte position from the least significant end
    if (le < len) {
      const uint64_t be = len - 1 - le;
      if (be < present) v |= (uint64_t)ld_byte(src + be) << (8 * j);
    }
  }
  return (uint32_t)(v >> (p & 7));
}

// bit i of the big-endian exponent of `len` bytes
MX_HD uint32_t exp_bit(const uint8_t* e, uint64_t len, uint64_t i) { return (ld_byte(e + len - 1 - (i >> 3)) >> (i & 7)) & 1u; }
// WIN-bit digit starting at bit i (a multiple of WIN; WIN = 4 never straddles a byte)
MX_HD uint32_t exp_digit(const uint8_t* e, uint64_t len, uint64_t i) {
  static_assert(WIN == 4, "digits are nibbles");
  return (ld_byte(e + len - 1 - (i >> 3)) >> (i & 4)) & 15u;
}

MX_HD int clz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __clz(x);
#else
  return x ? __builtin_clz(x) : 32;
#endif
}
MX_HD int ctz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __ffs(x) - 1;
#else
  return __builtin_ctz(x);
#endif
}

// the TPI lanes of one call; g is this lane's index in the group. Groups of several lanes exist only on the device; the host
// branches serve the one-lane group (TPI = 1), whose operations are plain code.
template <int TPI>
struct Grp {
  uint32_t g, mask;
#if defined(__CUDA_ARCH__)
  __device__ __forceinline__ Grp() {
    const uint32_t lane = threadIdx.x & 31;
    g = lane & (TPI - 1);
    mask = TPI == 32 ? 0xFFFFFFFFu : (((1u << TPI) - 1) << (lane & ~(TPI - 1)));
  }
#else
  Grp() : g(0), mask(1) {}
#endif
  MX_HD uint32_t bcast(uint32_t v, int src) const {
    if constexpr (TPI == 1) return v;
#if defined(__CUDA_ARCH__)
    else return __shfl_sync(mask, v, src, TPI);
#else
    else return v;
#endif
  }
  // the value of lane g + 1 (0 for the last lane)
  MX_HD uint32_t from_next(uint32_t v) const {
    if constexpr (TPI == 1) return 0;
#if defined(__CUDA_ARCH__)
    else { const uint32_t x = __shfl_down_sync(mask, v, 1, TPI); return g == TPI - 1 ? 0u : x; }
#else
    else return 0;
#endif
  }
  // the value of lane g - 1 (0 for lane 0)
  MX_HD uint64_t from_prev(uint64_t v) const {
    if constexpr (TPI == 1) return 0;
#if defined(__CUDA_ARCH__)
    else { const uint64_t x = __shfl_up_sync(mask, v, 1, TPI); return g == 0 ? 0ull : x; }
#else
    else return 0;
#endif
  }
  // predicate bits of the group's lanes, lane 0 in bit 0
  MX_HD uint32_t ballot(bool p) const {
    if constexpr (TPI == 1) return p;
#if defined(__CUDA_ARCH__)
    else return (__ballot_sync(mask, p) & mask) >> (threadIdx.x & 31 & ~(TPI - 1));
#else
    else return p;
#endif
  }
  // the carry into this lane when lanes generate (gen) and propagate (prop: all limbs 0xFFFFFFFF, or 0 for a borrow) carries;
  // `top` receives the carry out of the last lane. gen and prop are exclusive in every lane.
  MX_HD uint32_t carry_in(bool gen, bool prop, uint32_t& top) const {
    const uint64_t G = ballot(gen), P = ballot(prop);
    const uint64_t C = (P + (G << 1)) ^ P;   // bit i: the carry into lane i
    top = (uint32_t)(C >> TPI) & 1u;
    return (uint32_t)(C >> g) & 1u;
  }
};

template <int LL, int TPI, class G = Grp<TPI>>
struct Arith {
  static constexpr int L = LL * TPI;

  MX_HD static void set_zero(uint32_t* a) {
#pragma unroll
    for (int i = 0; i < LL; i++) a[i] = 0;
  }
  MX_HD static void copy(uint32_t* d, const uint32_t* s) {
#pragma unroll
    for (int i = 0; i < LL; i++) d[i] = s[i];
  }
  MX_HD static bool all_ones(const uint32_t* a) {
    uint32_t x = 0xFFFFFFFFu;
#pragma unroll
    for (int i = 0; i < LL; i++) x &= a[i];
    return x == 0xFFFFFFFFu;
  }
  MX_HD static bool lane_zero(const uint32_t* a) {
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < LL; i++) x |= a[i];
    return x == 0;
  }
  MX_HD static bool is_zero(const G& g, const uint32_t* a) { return g.ballot(!lane_zero(a)) == 0; }
  // a += c (a 64-bit value at limb 0); returns the carry out of the lane
  MX_HD static uint32_t add_small(uint32_t* a, uint64_t c) {
    uint64_t s = (uint64_t)a[0] + (uint32_t)c;
    a[0] = (uint32_t)s;
    s = (s >> 32) + (uint64_t)a[1] + (c >> 32);
    a[1] = (uint32_t)s;
#pragma unroll
    for (int i = 2; i < LL; i++) {
      s = (s >> 32) + a[i];
      a[i] = (uint32_t)s;
    }
    return (uint32_t)(s >> 32);
  }
  // a -= c (c in {0, 1}); returns the borrow out of the lane
  MX_HD static uint32_t sub_bit(uint32_t* a, uint32_t c) {
    uint32_t br = c;
#pragma unroll
    for (int i = 0; i < LL; i++) {
      const uint32_t x = a[i];
      a[i] = x - br;
      br = br & (x == 0);
    }
    return br;
  }
  // r = a + b over the whole group; returns the carry out of the top limb
  MX_HD static uint32_t add(const G& g, uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint64_t s = 0;
#pragma unroll
    for (int i = 0; i < LL; i++) {
      s = (s >> 32) + a[i] + b[i];
      r[i] = (uint32_t)s;
    }
    const bool gen = (s >> 32) != 0;
    uint32_t top;
    const uint32_t cin = g.carry_in(gen, !gen && all_ones(r), top);
    add_small(r, cin);
    return top;
  }
  // r = a - b over the whole group; returns the borrow out of the top limb
  MX_HD static uint32_t sub(const G& g, uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t br = 0;
#pragma unroll
    for (int i = 0; i < LL; i++) {
      const uint64_t d = (uint64_t)a[i] - b[i] - br;
      r[i] = (uint32_t)d;
      br = (uint32_t)(d >> 63);
    }
    uint32_t top;
    const uint32_t bin = g.carry_in(br != 0, br == 0 && lane_zero(r), top);
    sub_bit(r, bin);
    return top;
  }
  // a >= q for the group's value a (group-wide compare from the most significant lane that differs)
  MX_HD static bool geq(const G& g, const uint32_t* a, const uint32_t* q) {
    int c = 0;   // this lane: +1 a > q, -1 a < q, 0 equal
#pragma unroll
    for (int i = LL - 1; i >= 0; i--)
      if (c == 0) c = a[i] > q[i] ? 1 : (a[i] < q[i] ? -1 : 0);
    const uint32_t gt = g.ballot(c > 0), lt = g.ballot(c < 0);
    const uint32_t any = gt | lt;
    if (any == 0) return true;
    return (gt >> (31 - clz32(any))) & 1u;
  }
  // a = a - q when force or a >= q
  MX_HD static void cond_sub(const G& g, uint32_t* a, const uint32_t* q, bool force) {
    if (force || geq(g, a, q)) sub(g, a, a, q);
  }
  // r = a + b mod q for a, b < q
  MX_HD static void add_mod(const G& g, uint32_t* r, const uint32_t* a, const uint32_t* b, const uint32_t* q) {
    const uint32_t top = add(g, r, a, b);
    cond_sub(g, r, q, top != 0);
  }

  // The shifting accumulator of both products: t (LL limbs per lane) and th, the lane's carry word at limb LL.
  // One step adds a b_j, and with REDC m q (m = t_0 m0'); then shifts right by one limb. Returns the limb shifted out (exact:
  // lane 0 has no pending carries below it).
  template <bool REDC>
  MX_HD static uint32_t step(const G& g, uint32_t* t, uint64_t& th, const uint32_t* a, uint32_t bj, const uint32_t* q, uint32_t m0) {
    uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < LL; i++) {
      c = (uint64_t)a[i] * bj + t[i] + (c >> 32);
      t[i] = (uint32_t)c;
    }
    th += c >> 32;
    if constexpr (REDC) {
      const uint32_t m = g.bcast(t[0] * m0, 0);
      c = 0;
#pragma unroll
      for (int i = 0; i < LL; i++) {
        c = (uint64_t)q[i] * m + t[i] + (c >> 32);
        t[i] = (uint32_t)c;
      }
      th += c >> 32;
    }
    const uint32_t out = g.bcast(t[0], 0);
    const uint32_t nxt = g.from_next(t[0]);
#pragma unroll
    for (int i = 0; i < LL - 1; i++) t[i] = t[i + 1];
    th += nxt;
    t[LL - 1] = (uint32_t)th;
    th >>= 32;
    return out;
  }

  // r = a b R^-1 mod q (a < R, b < q, q odd; r < q). r may alias a or b.
  MX_HD static void mont_mul(const G& g, uint32_t* r, const uint32_t* a, const uint32_t* b, const uint32_t* q, uint32_t m0) {
    uint32_t t[LL], bb[LL];
    uint64_t th = 0;
    copy(bb, b);
    set_zero(t);
#pragma unroll 1
    for (int jj = 0; jj < TPI; jj++) {
#pragma unroll
      for (int w = 0; w < LL; w++) step<true>(g, t, th, a, g.bcast(bb[w], jj), q, m0);
    }
    // resolve: each lane's carry word joins the next lane's limb 0; the last lane's is the top word (t < 2q < 2^(32L + 1))
    const uint64_t cprev = g.from_prev(th);
    const uint32_t gen = add_small(t, cprev);
    uint32_t top;
    const uint32_t cin = g.carry_in(gen != 0, gen == 0 && all_ones(t), top);
    add_small(t, cin);
    const uint32_t hi = (uint32_t)g.bcast((uint32_t)th, TPI - 1) + top;
    copy(r, t);
    cond_sub(g, r, q, hi != 0);
  }

  // r = a b mod 2^(32 L) (the low half). r may alias a or b.
  MX_HD static void mul_lo(const G& g, uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t t[LL], bb[LL], lo[LL];
    uint64_t th = 0;
    copy(bb, b);
    set_zero(t);
#pragma unroll 1
    for (int jj = 0; jj < TPI; jj++) {
#pragma unroll
      for (int w = 0; w < LL; w++) {
        const uint32_t o = step<false>(g, t, th, a, g.bcast(bb[w], jj), nullptr, 0);
        if (g.g == (uint32_t)jj) lo[w] = o;
      }
    }
    copy(r, lo);
  }

  // a mod 2^k
  MX_HD static void mask_bits(const G& g, uint32_t* a, uint32_t k) {
#pragma unroll
    for (int i = 0; i < LL; i++) {
      const uint32_t base = 32 * (g.g * LL + i);
      if (base >= k) a[i] = 0;
      else if (k - base < 32) a[i] &= (1u << (k - base)) - 1;
    }
  }

  // trailing zeros of the group's value (32 L for zero)
  MX_HD static uint32_t tzeros(const G& g, const uint32_t* a) {
    uint32_t v = 0xFFFFFFFFu;   // this lane's count, from its lowest non-zero limb
#pragma unroll
    for (int i = LL - 1; i >= 0; i--)
      if (a[i]) v = 32 * (g.g * LL + i) + ctz32(a[i]);
    const uint32_t nz = g.ballot(v != 0xFFFFFFFFu);
    if (nz == 0) return 32 * L;
    return g.bcast(v, ctz32(nz));
  }

  // ---- the odd part --------------------------------------------------------------------------------------------------------
  // R^2 mod q from 2^(bits(q) - 1) < q: (32 L + 2 - bits(q)) doublings give 2^(32 L + 1) = Mont(2), then log2(32 L) Montgomery
  // squarings Mont(2^e) -> Mont(2^2e) reach Mont(2^(32 L)) = R^2 mod q. q >= 3.
  MX_HD static void r2_mod(const G& g, uint32_t* x, const uint32_t* q, uint32_t qbits, uint32_t m0) {
    set_zero(x);
    const uint32_t tb = qbits - 1;
    if (tb / 32 / LL == g.g) {
#pragma unroll
      for (int i = 0; i < LL; i++)
        if ((uint32_t)i == (tb / 32) % LL) x[i] = 1u << (tb & 31);
    }
#pragma unroll 1
    for (uint32_t d = 0; d < 32 * L + 2 - qbits; d++) add_mod(g, x, x, x, q);
#pragma unroll 1
    for (uint32_t s = 1; s < 32 * (uint32_t)L; s <<= 1) mont_mul(g, x, x, x, q, m0);
  }

  // -q^-1 mod 2^32 (q odd) by Newton iteration
  MX_HD static uint32_t neg_inv32(uint32_t q0) {
    uint32_t x = q0;   // q0 q0 = 1 mod 8
#pragma unroll
    for (int i = 0; i < 4; i++) x *= 2u - q0 * x;
    return 0u - x;
  }

  // the shared-memory table: entry d (1..TAB), limb i of this lane at tab[((d - 1) LL + i) stride]
  MX_HD static void tab_store(uint32_t* tab, int stride, int d, const uint32_t* a) {
#pragma unroll
    for (int i = 0; i < LL; i++) tab[((d - 1) * LL + i) * stride] = a[i];
  }
  MX_HD static void tab_load(const uint32_t* tab, int stride, int d, uint32_t* a) {
#pragma unroll
    for (int i = 0; i < LL; i++) a[i] = tab[((d - 1) * LL + i) * stride];
  }

  // a1 = b^e mod q (q odd, >= 3)
  MX_HD static void pow_odd(const G& g, uint32_t* a1, const uint8_t* in, const Desc& d, const uint32_t* q, uint32_t qbits,
                            uint32_t* tab, int stride) {
    const uint32_t m0 = neg_inv32(g.bcast(q[0], 0));
    uint32_t r2[LL], x[LL], c[LL];
    r2_mod(g, r2, q, qbits, m0);
    // base: from the most significant L-limb chunk down, x <- MM(x, R^2) + MM(c_j, R^2) = Mont(x R + c_j)
    const uint64_t chunks = (d.b_len + 4 * L - 1) / (4 * L);
#pragma unroll 1
    for (uint64_t j = chunks; j-- > 0;) {
#pragma unroll
      for (int i = 0; i < LL; i++) c[i] = load_word(in + d.b_off, d.b_len, d.b_len, 32 * (uint64_t)L * j, g.g * LL + i);
      mont_mul(g, c, c, r2, q, m0);
      if (j + 1 == chunks) {
        copy(x, c);
      } else {
        mont_mul(g, x, x, r2, q, m0);
        add_mod(g, x, x, c, q);
      }
    }
    // the table Mont(b^1 .. b^15)
    tab_store(tab, stride, 1, x);
    copy(c, x);
#pragma unroll 1
    for (int e = 2; e <= TAB; e++) {
      mont_mul(g, c, c, x, q, m0);
      tab_store(tab, stride, e, c);
    }
    // fixed window, most significant digit first
    const uint64_t nwin = (d.e_bits + WIN - 1) / WIN;
    const uint8_t* e = in + d.e_off;
    tab_load(tab, stride, (int)exp_digit(e, d.e_len, WIN * (nwin - 1)), x);   // the top digit is not zero
#pragma unroll 1
    for (uint64_t w = nwin - 1; w-- > 0;) {
#pragma unroll 1
      for (int s = 0; s < WIN; s++) mont_mul(g, x, x, x, q, m0);
      const uint32_t dg = exp_digit(e, d.e_len, WIN * w);
      if (dg) {
        tab_load(tab, stride, (int)dg, c);
        mont_mul(g, x, x, c, q, m0);
      }
    }
    // out of Montgomery form: MM(x, 1)
    set_zero(c);
    if (g.g == 0) c[0] = 1;
    mont_mul(g, a1, x, c, q, m0);
  }

  // ---- the power-of-two part -----------------------------------------------------------------------------------------------
  // a2 = b^e mod 2^k (1 <= k <= 32 L), MSB-first square-and-multiply on truncated products. For odd b only the low k - 1
  // exponent bits matter (b^(2^(k-1)) = 1 mod 2^k); for even b with tz(b) + msb(e) >= k the result is 0. At most k squarings.
  MX_HD static void pow_2k(const G& g, uint32_t* a2, const uint8_t* in, const Desc& d, uint32_t k) {
    uint32_t b[LL];
#pragma unroll
    for (int i = 0; i < LL; i++) b[i] = load_word(in + d.b_off, d.b_len, d.b_len, 0, g.g * LL + i);
    mask_bits(g, b, k);
    set_zero(a2);
    if (is_zero(g, b)) return;                 // b = 0 mod 2^k, e >= 1
    const uint64_t msb = d.e_bits - 1;
    uint64_t nb;
    if (g.bcast(b[0], 0) & 1u) {
      nb = msb + 1 < (uint64_t)k - 1 ? msb + 1 : (uint64_t)k - 1;
    } else {
      if ((uint64_t)tzeros(g, b) + msb >= k) return;
      nb = msb + 1;
    }
    if (g.g == 0) a2[0] = 1;
    const uint8_t* e = in + d.e_off;
#pragma unroll 1
    for (uint64_t i = nb; i-- > 0;) {
      mul_lo(g, a2, a2, a2);
      if (exp_bit(e, d.e_len, i)) mul_lo(g, a2, a2, b);
      mask_bits(g, a2, k);
    }
  }

  // ---- one call --------------------------------------------------------------------------------------------------------------
  // r = b^e mod M, M >= 2, e >= 1
  MX_HD static void run(const G& g, uint32_t* r, const uint8_t* in, const Desc& d, uint32_t* tab, int stride) {
    const uint32_t k = (uint32_t)d.k, qbits = (uint32_t)(d.m_bits - d.k);
    uint32_t q[LL], a1[LL];
#pragma unroll
    for (int i = 0; i < LL; i++) q[i] = load_word(in + d.m_off, d.m_len, d.m_present, k, g.g * LL + i);
    if (qbits >= 2) pow_odd(g, a1, in, d, q, qbits, tab, stride);
    if (k == 0) { copy(r, a1); return; }
    pow_2k(g, r, in, d, k);
    if (qbits < 2) return;                     // M = 2^k
    // CRT: y = (a2 - a1) q^-1 mod 2^k, r = a1 + q y < M
    uint32_t x[LL], t[LL];
    set_zero(x);
    if (g.g == 0) x[0] = 0u - neg_inv32(q[0]);   // q^-1 mod 2^32
#pragma unroll 1
    for (int bits = 32; bits < 32 * L; bits *= 2) {  // x <- x (2 - q x) mod 2^(32 L): correct bits double
      mul_lo(g, t, q, x);
      uint32_t two[LL];
      set_zero(two);
      if (g.g == 0) two[0] = 2;
      sub(g, t, two, t);
      mul_lo(g, x, x, t);
    }
    sub(g, t, r, a1);                          // a2 - a1 mod 2^(32 L)
    mask_bits(g, t, k);
    mul_lo(g, t, t, x);
    mask_bits(g, t, k);
    mul_lo(g, t, q, t);
    add(g, r, t, a1);
  }

  // r (the group's L limbs) as 4 L big-endian bytes at out (4-byte aligned)
  MX_HD static void store_be(const G& g, uint8_t* out, const uint32_t* r) {
#pragma unroll
    for (int i = 0; i < LL; i++) {
      const uint32_t gw = g.g * LL + i, w = r[i];
      uint32_t be = (w >> 24) | ((w >> 8) & 0xFF00u) | ((w << 8) & 0xFF0000u) | (w << 24);
      *reinterpret_cast<uint32_t*>(out + 4 * (L - 1 - gw)) = be;
    }
  }
};

}  // namespace modexp
}  // namespace b200
