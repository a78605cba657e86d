// Host-side (CPU) field / point arithmetic used by the product's serial tail.
//
// The device produces one bucket-sum point per window; combining W <= ~40 window sums is an inherently serial
// chain of ~bits doublings (r = 2^c * r + S_w).  One GPU thread takes an order of magnitude longer per doubling than a host core,
// so this tail -- and only this tail -- runs on the calling host thread (see DESIGN.md "serial tail").
// It is part of the product, not the oracle: there is no alternative CPU path for the bucket work.
//
// Follows the same value conventions as the reference (Montgomery residues, R = 2^(64*limbs);
// reference constantine/math/arithmetic/limbs_montgomery.nim:180-217 for CIOS), written for
// 64-bit limbs with unsigned __int128.
#pragma once
#include <chrono>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include "field_constants.cuh"

#if defined(__x86_64__) && defined(__GNUC__)
#include <cpuid.h>
#define B200_HOST_MULX_ADX 1
#endif

namespace b200 {
namespace host {

typedef unsigned __int128 u128;

#if defined(B200_HOST_MULX_ADX)
// x86-64 with BMI2 + ADX: the same CIOS multiplication with MULX and the two independent carry chains of
// ADCX (CF) / ADOX (OF) -- about half the time of the portable form, and the host tail is ~3000 dependent multiplications per MSM.
// Chosen at run time (CPUID leaf 7: EBX bit 8 = BMI2, bit 19 = ADX), the library is built on another machine.
// `-DB200_HOST_PORTABLE_MUL` or the environment variable CTT_B200_HOST_PORTABLE_MUL=1 keeps the portable form.
inline bool cpu_has_mulx_adx() {
  static const bool v = [] {
#if defined(B200_HOST_PORTABLE_MUL)
    return false;
#else
    const char* e = getenv("CTT_B200_HOST_PORTABLE_MUL");
    if (e && e[0] == '1') return false;
    unsigned a = 0, b = 0, c = 0, d = 0;
    if (!__get_cpuid_count(7, 0, &a, &b, &c, &d)) return false;
    return ((b >> 8) & 1u) && ((b >> 19) & 1u);
#endif
  }();
  return v;
}

// One row: (t0 .. t_N, carry into t_{N+1}) += x[0 .. N-1] * y.  Low halves ride the OF chain into t_j, high halves the CF chain into
// t_{j+1}; the two final carries land in t_N / t_{N+1}.
#define B200_MULX_STEP(off, lo, hi) "mulx " #off "(%[x]), %%r8, %%r9\n\t" "adox %%r8, %[" #lo "]\n\t" "adcx %%r9, %[" #hi "]\n\t"
inline void mulx_row6(uint64_t& t0, uint64_t& t1, uint64_t& t2, uint64_t& t3, uint64_t& t4, uint64_t& t5, uint64_t& t6, uint64_t& t7,
                      const uint64_t* x, uint64_t y) {
  __asm__ volatile(
      "xorl %%eax, %%eax\n\t"   // CF = OF = 0
      B200_MULX_STEP(0, a0, a1) B200_MULX_STEP(8, a1, a2) B200_MULX_STEP(16, a2, a3)
      B200_MULX_STEP(24, a3, a4) B200_MULX_STEP(32, a4, a5) B200_MULX_STEP(40, a5, a6)
      "movl $0, %%r8d\n\t" "adox %%r8, %[a6]\n\t" "adcx %%r8, %[a7]\n\t" "adox %%r8, %[a7]\n\t"
      : [a0] "+r"(t0), [a1] "+r"(t1), [a2] "+r"(t2), [a3] "+r"(t3), [a4] "+r"(t4), [a5] "+r"(t5), [a6] "+r"(t6), [a7] "+r"(t7)
      : [x] "r"(x), "d"(y)
      : "rax", "r8", "r9", "cc", "memory");
}
inline void mulx_row4(uint64_t& t0, uint64_t& t1, uint64_t& t2, uint64_t& t3, uint64_t& t4, uint64_t& t5, const uint64_t* x, uint64_t y) {
  __asm__ volatile(
      "xorl %%eax, %%eax\n\t"
      B200_MULX_STEP(0, a0, a1) B200_MULX_STEP(8, a1, a2) B200_MULX_STEP(16, a2, a3) B200_MULX_STEP(24, a3, a4)
      "movl $0, %%r8d\n\t" "adox %%r8, %[a4]\n\t" "adcx %%r8, %[a5]\n\t" "adox %%r8, %[a5]\n\t"
      : [a0] "+r"(t0), [a1] "+r"(t1), [a2] "+r"(t2), [a3] "+r"(t3), [a4] "+r"(t4), [a5] "+r"(t5)
      : [x] "r"(x), "d"(y)
      : "rax", "r8", "r9", "cc", "memory");
}
#undef B200_MULX_STEP
#endif

template <class F>
struct HFp {
  static constexpr int N = F::N64;
  uint64_t l[N];

  static HFp zero() { HFp r; for (int i = 0; i < N; i++) r.l[i] = 0; return r; }
  static HFp one() { HFp r; for (int i = 0; i < N; i++) r.l[i] = F::ONE64(i); return r; }
  bool is_zero() const { uint64_t o = 0; for (int i = 0; i < N; i++) o |= l[i]; return o == 0; }
  bool operator==(const HFp& b) const { uint64_t o = 0; for (int i = 0; i < N; i++) o |= l[i] ^ b.l[i]; return o == 0; }

  static bool geq_p(const uint64_t* a) {
    for (int i = N - 1; i >= 0; i--) {
      if (a[i] > F::P64(i)) return true;
      if (a[i] < F::P64(i)) return false;
    }
    return true;
  }
  static void sub_p(uint64_t* a) {
    u128 borrow = 0;
    for (int i = 0; i < N; i++) {
      u128 d = (u128)a[i] - F::P64(i) - borrow;
      a[i] = (uint64_t)d;
      borrow = (d >> 64) & 1;
    }
  }
  HFp operator+(const HFp& b) const {
    HFp r; u128 c = 0;
    for (int i = 0; i < N; i++) { c += (u128)l[i] + b.l[i]; r.l[i] = (uint64_t)c; c >>= 64; }
    if (c || geq_p(r.l)) sub_p(r.l);
    return r;
  }
  HFp operator-(const HFp& b) const {
    HFp r; u128 borrow = 0;
    for (int i = 0; i < N; i++) {
      u128 d = (u128)l[i] - b.l[i] - borrow;
      r.l[i] = (uint64_t)d;
      borrow = (d >> 64) & 1;
    }
    if (borrow) {
      u128 c = 0;
      for (int i = 0; i < N; i++) { c += (u128)r.l[i] + F::P64(i); r.l[i] = (uint64_t)c; c >>= 64; }
    }
    return r;
  }
  // the modulus as an array (MULX takes its multiplicand from memory)
  static const uint64_t* modulus() {
    static const struct M { uint64_t v[N]; M() { for (int i = 0; i < N; i++) v[i] = F::P64(i); } } m;
    return m.v;
  }
  HFp operator*(const HFp& b) const {
#if defined(B200_HOST_MULX_ADX)
    if ((N == 6 || N == 4) && cpu_has_mulx_adx()) return mul_mulx_adx(b);
#endif
    return mul_portable(b);
  }
#if defined(B200_HOST_MULX_ADX)
  HFp mul_mulx_adx(const HFp& b) const {
    const uint64_t* p = modulus();
    HFp r;
    uint64_t carry;
    if constexpr (N == 6) {
      uint64_t t0 = 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0, t5 = 0, t6 = 0, t7 = 0;
      // a row of a * b_i, a row of m * p that clears the lowest limb, and the window slides up one limb: instead of moving eight
      // registers the NAMES rotate (the cleared limb becomes the new top limb)
#define B200_CIOS6(a0, a1, a2, a3, a4, a5, a6, a7, i) \
  mulx_row6(a0, a1, a2, a3, a4, a5, a6, a7, l, b.l[i]); mulx_row6(a0, a1, a2, a3, a4, a5, a6, a7, p, a0 * F::INV64); a0 = 0;
      B200_CIOS6(t0, t1, t2, t3, t4, t5, t6, t7, 0)
      B200_CIOS6(t1, t2, t3, t4, t5, t6, t7, t0, 1)
      B200_CIOS6(t2, t3, t4, t5, t6, t7, t0, t1, 2)
      B200_CIOS6(t3, t4, t5, t6, t7, t0, t1, t2, 3)
      B200_CIOS6(t4, t5, t6, t7, t0, t1, t2, t3, 4)
      B200_CIOS6(t5, t6, t7, t0, t1, t2, t3, t4, 5)
#undef B200_CIOS6
      r.l[0] = t6; r.l[1] = t7; r.l[2] = t0; r.l[3] = t1; r.l[4] = t2; r.l[5] = t3;
      carry = t4;
    } else if constexpr (N == 4) {
      uint64_t t0 = 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0, t5 = 0;
#define B200_CIOS4(a0, a1, a2, a3, a4, a5, i) \
  mulx_row4(a0, a1, a2, a3, a4, a5, l, b.l[i]); mulx_row4(a0, a1, a2, a3, a4, a5, p, a0 * F::INV64); a0 = 0;
      B200_CIOS4(t0, t1, t2, t3, t4, t5, 0)
      B200_CIOS4(t1, t2, t3, t4, t5, t0, 1)
      B200_CIOS4(t2, t3, t4, t5, t0, t1, 2)
      B200_CIOS4(t3, t4, t5, t0, t1, t2, 3)
#undef B200_CIOS4
      r.l[0] = t4; r.l[1] = t5; r.l[2] = t0; r.l[3] = t1;
      carry = t2;
    } else {
      return mul_portable(b);
    }
    if (carry || geq_p(r.l)) sub_p(r.l);
    return r;
  }
#endif
  HFp mul_portable(const HFp& b) const {
    uint64_t t[N + 2];
    for (int i = 0; i < N + 2; i++) t[i] = 0;
    for (int i = 0; i < N; i++) {
      u128 c = 0;
      for (int j = 0; j < N; j++) {
        c += (u128)l[j] * b.l[i] + t[j];
        t[j] = (uint64_t)c; c >>= 64;
      }
      c += t[N]; t[N] = (uint64_t)c; t[N + 1] = (uint64_t)(c >> 64);
      uint64_t m = t[0] * F::INV64;
      c = (u128)m * F::P64(0) + t[0];
      c >>= 64;
      for (int j = 1; j < N; j++) {
        c += (u128)m * F::P64(j) + t[j];
        t[j - 1] = (uint64_t)c; c >>= 64;
      }
      c += t[N]; t[N - 1] = (uint64_t)c; c >>= 64;
      t[N] = t[N + 1] + (uint64_t)c;
    }
    HFp r;
    for (int i = 0; i < N; i++) r.l[i] = t[i];
    if (t[N] || geq_p(r.l)) sub_p(r.l);
    return r;
  }
  HFp sqr() const { return (*this) * (*this); }
  HFp dbl() const { return (*this) + (*this); }
  HFp neg() const { if (is_zero()) return *this; return zero() - *this; }
  // a^(p-2) (Fermat); only used off the hot path (test/bench input generation, affine normalisation helpers)
  HFp inv() const {
    uint64_t e[N];
    for (int i = 0; i < N; i++) e[i] = F::P64(i);
    e[0] -= 2;  // p is odd and > 2: no borrow
    HFp r = one(), b = *this;
    for (int i = 0; i < 64 * N; i++) {
      if ((e[i >> 6] >> (i & 63)) & 1) r = r * b;
      b = b.sqr();
    }
    return r;
  }
};

template <class F>
struct HFp2 {
  typedef HFp<F> Base;
  Base c0, c1;
  static HFp2 zero() { HFp2 r; r.c0 = Base::zero(); r.c1 = Base::zero(); return r; }
  static HFp2 one() { HFp2 r; r.c0 = Base::one(); r.c1 = Base::zero(); return r; }
  bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  bool operator==(const HFp2& b) const { return c0 == b.c0 && c1 == b.c1; }
  HFp2 operator+(const HFp2& b) const { HFp2 r; r.c0 = c0 + b.c0; r.c1 = c1 + b.c1; return r; }
  HFp2 operator-(const HFp2& b) const { HFp2 r; r.c0 = c0 - b.c0; r.c1 = c1 - b.c1; return r; }
  HFp2 operator*(const HFp2& b) const {
    Base v0 = c0 * b.c0, v1 = c1 * b.c1, s = (c0 + c1) * (b.c0 + b.c1);
    HFp2 r; r.c0 = v0 - v1; r.c1 = (s - v0) - v1; return r;
  }
  HFp2 sqr() const { Base t = c0 * c1; HFp2 r; r.c0 = (c0 + c1) * (c0 - c1); r.c1 = t + t; return r; }
  HFp2 dbl() const { HFp2 r; r.c0 = c0.dbl(); r.c1 = c1.dbl(); return r; }
  HFp2 neg() const { HFp2 r; r.c0 = c0.neg(); r.c1 = c1.neg(); return r; }
  HFp2 inv() const {
    Base n = (c0.sqr() + c1.sqr()).inv();
    HFp2 r; r.c0 = c0 * n; r.c1 = (c1 * n).neg(); return r;
  }
};

// Extended-Jacobian ("XYZZ") point: x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2; infinity iff ZZ == 0.
// Same coordinate system the device buckets use (formulas: EFD shortw "xyzz", add-2008-s / dbl-2008-s-1, a = 0;
// the reference carries the same system in constantine/math/elliptic/ec_shortweierstrass_jacobian_extended.nim:30-40).
template <class T>
struct HXyzz {
  T x, y, zz, zzz;
  static HXyzz inf() { HXyzz r; r.x = T::zero(); r.y = T::zero(); r.zz = T::zero(); r.zzz = T::zero(); return r; }
  bool is_inf() const { return zz.is_zero(); }
};

template <class T>
inline HXyzz<T> xyzz_dbl(const HXyzz<T>& p) {
  if (p.is_inf()) return p;
  T U = p.y.dbl();
  T V = U.sqr();
  T W = U * V;
  T S = p.x * V;
  T X2 = p.x.sqr();
  T M = X2.dbl() + X2;
  HXyzz<T> r;
  r.x = M.sqr() - S.dbl();
  r.y = M * (S - r.x) - W * p.y;
  r.zz = V * p.zz;
  r.zzz = W * p.zzz;
  return r;
}

template <class T>
inline HXyzz<T> xyzz_add(const HXyzz<T>& p, const HXyzz<T>& q) {
  if (p.is_inf()) return q;
  if (q.is_inf()) return p;
  T U1 = p.x * q.zz, U2 = q.x * p.zz;
  T S1 = p.y * q.zzz, S2 = q.y * p.zzz;
  T P = U2 - U1, R = S2 - S1;
  if (P.is_zero()) {
    if (R.is_zero()) return xyzz_dbl(p);
    return HXyzz<T>::inf();
  }
  T PP = P.sqr();
  T PPP = P * PP;
  T Q = U1 * PP;
  HXyzz<T> r;
  r.x = R.sqr() - PPP - Q.dbl();
  r.y = R * (Q - r.x) - S1 * PPP;
  r.zz = p.zz * q.zz * PP;
  r.zzz = p.zzz * q.zzz * PPP;
  return r;
}

// XYZZ -> Jacobian (X, Y, Z) with x = X/Z^2, y = Y/Z^3, no inversion:  Z := ZZ*ZZZ  (Z^2 = ZZ^2 ZZZ^2, Z^3 = ZZ^3 ZZZ^3)
//   X = x Z^2 = X1 * ZZ * ZZZ^2 ;  Y = y Z^3 = Y1 * ZZ^3 * ZZZ^2.
// Infinity is written as (1, 1, 0) like the reference does (ec_shortweierstrass_jacobian.nim:46-63).
template <class T>
inline void xyzz_to_jac(const HXyzz<T>& p, T& X, T& Y, T& Z) {
  if (p.is_inf()) { X = T::one(); Y = T::one(); Z = T::zero(); return; }
  T zzz2 = p.zzz.sqr();
  T zz2 = p.zz.sqr();
  X = p.x * p.zz * zzz2;
  Y = p.y * zz2 * p.zz * zzz2;
  Z = p.zz * p.zzz;
}

// XYZZ -> homogeneous projective (X, Y, Z) with x = X/Z, y = Y/Z:  Z := ZZ*ZZZ, X = X1*ZZZ, Y = Y1*ZZ.
// Infinity is (0, 1, 0) (reference ec_shortweierstrass_projective.nim:46-62).
template <class T>
inline void xyzz_to_prj(const HXyzz<T>& p, T& X, T& Y, T& Z) {
  if (p.is_inf()) { X = T::zero(); Y = T::one(); Z = T::zero(); return; }
  X = p.x * p.zzz;
  Y = p.y * p.zz;
  Z = p.zz * p.zzz;
}

}  // namespace host

// milliseconds on the host clock since t0, for the entries' last_timing splits
inline double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace b200
