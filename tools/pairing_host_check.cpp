// The host pairing (constantine_b200/csrc/host_pairing.hpp) and the cell-batch challenge (eth_kzg_host.hpp) behind a line protocol, so
// that the CPU suite can check them (tests/test_peerdas_verify_host.py builds this with the host compiler). Points are compressed hex.
//   g2 <hex96>                  -> "<status> <recompressed hex96 or ->" (decode, curve and subgroup check)
//   mul1 <hex48> <k> / mul2 <hex96> <k>   -> [k]P compressed; k is 32 bytes big-endian (hex)
//   add1 <hex48> <hex48>        -> P1 + P2 compressed
//   neg1 <hex48>                -> -P compressed
//   eq <P1> <Q1> <P2> <Q2>      -> 1 if e(P1, Q1) == e(P2, Q2), else 0
//   one <P> <Q>                 -> 1 if e(P, Q) == 1, else 0
//   check <P1> <Q1> <P2> <Q2>   -> pairing_check: 1 if e(P1, Q1) e(P2, Q2) == 1, else 0
//   challenge <U> <commitments (U x 48 bytes, "-" if none)> <n>, then n lines "<commitment idx> <cell idx> <cell> <proof>"
//                               -> the verify_cell_kzg_proof_batch challenge, 32 bytes big-endian
#include <cstdio>
#include <iostream>
#include <string>
#include <vector>
#include "eth_kzg_host.hpp"
#include "host_pairing.hpp"

using namespace b200;
using namespace b200::bls12_381;

static std::vector<uint8_t> unhex(const std::string& s) {
  std::vector<uint8_t> v;
  if (s == "-") return v;
  for (size_t i = 0; i + 1 < s.size(); i += 2) v.push_back((uint8_t)std::stoi(s.substr(i, 2), nullptr, 16));
  return v;
}
static std::string hex(const uint8_t* p, size_t n) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (size_t i = 0; i < n; i++) { s += d[p[i] >> 4]; s += d[p[i] & 15]; }
  return s;
}

template <class T>
static host::HXyzz<T> to_xyzz(const T& x, const T& y) {
  if (x.is_zero() && y.is_zero()) return host::HXyzz<T>::inf();
  host::HXyzz<T> p; p.x = x; p.y = y; p.zz = T::one(); p.zzz = T::one();
  return p;
}
template <class T>
static void to_affine(const host::HXyzz<T>& p, T& x, T& y) {
  if (p.is_inf()) { x = T::zero(); y = T::zero(); return; }
  x = p.x * p.zz.inv(); y = p.y * p.zzz.inv();
}
template <class T>
static host::HXyzz<T> scalar_mul(const host::HXyzz<T>& p, const uint8_t k[32]) {
  host::HXyzz<T> acc = host::HXyzz<T>::inf();
  for (int i = 0; i < 256; i++) {
    acc = host::xyzz_dbl(acc);
    if ((k[i >> 3] >> (7 - (i & 7))) & 1) acc = host::xyzz_add(acc, p);
  }
  return acc;
}

static G1Aff g1(const std::string& h) {
  const std::vector<uint8_t> b = unhex(h);
  G1Aff p;
  if (b.size() != 48 || decompress_g1(p.x, p.y, b.data()) != Success) { fprintf(stderr, "bad G1 %s\n", h.c_str()); exit(2); }
  return p;
}
static G2Aff g2(const std::string& h) {
  const std::vector<uint8_t> b = unhex(h);
  G2Aff q;
  if (b.size() != 96 || decompress_g2(q, b.data()) != Success) { fprintf(stderr, "bad G2 %s\n", h.c_str()); exit(2); }
  return q;
}
static std::string out1(const host::HXyzz<Fp>& p) {
  G1Aff a; to_affine(p, a.x, a.y);
  uint8_t o[48]; compress_g1(o, a.x, a.y, p.is_inf());
  return hex(o, 48);
}
static std::string out2(const host::HXyzz<Fp2>& p) {
  G2Aff a; to_affine(p, a.x, a.y);
  uint8_t o[96]; compress_g2(o, a);
  return hex(o, 96);
}

int main() {
  std::string cmd;
  while (std::cin >> cmd) {
    if (cmd == "g2") {
      std::string a; std::cin >> a;
      const std::vector<uint8_t> b = unhex(a);
      G2Aff q;
      const int st = b.size() == 96 ? check_g2(q, b.data()) : -1;
      std::string re = "-";
      if (st == Success) { uint8_t o[96]; compress_g2(o, q); re = hex(o, 96); }
      std::cout << st << " " << re << "\n";
    } else if (cmd == "mul1" || cmd == "mul2") {
      std::string a, k; std::cin >> a >> k;
      const std::vector<uint8_t> kb = unhex(k);
      if (cmd == "mul1") { const G1Aff p = g1(a); std::cout << out1(scalar_mul(to_xyzz(p.x, p.y), kb.data())) << "\n"; }
      else { const G2Aff q = g2(a); std::cout << out2(scalar_mul(to_xyzz(q.x, q.y), kb.data())) << "\n"; }
    } else if (cmd == "add1" || cmd == "neg1") {
      std::string a, b; std::cin >> a;
      const G1Aff p = g1(a);
      if (cmd == "neg1") { std::cout << out1(to_xyzz(p.x, p.y.neg())) << "\n"; continue; }
      std::cin >> b;
      const G1Aff q = g1(b);
      std::cout << out1(host::xyzz_add(to_xyzz(p.x, p.y), to_xyzz(q.x, q.y))) << "\n";
    } else if (cmd == "eq" || cmd == "check") {
      std::string a, b, c, d; std::cin >> a >> b >> c >> d;
      const G1Aff p1 = g1(a), p2 = g1(c);
      const G2Aff q1 = g2(b), q2 = g2(d);
      if (cmd == "eq") std::cout << (pairing(p1, q1) == pairing(p2, q2) ? 1 : 0) << "\n";
      else std::cout << (pairing_check(p1, q1, p2, q2) ? 1 : 0) << "\n";
    } else if (cmd == "one") {
      std::string a, b; std::cin >> a >> b;
      std::cout << (pairing(g1(a), g2(b)).is_one() ? 1 : 0) << "\n";
    } else if (cmd == "challenge") {
      size_t u = 0, n = 0;
      std::string cm;
      std::cin >> u >> cm >> n;
      const std::vector<uint8_t> commitments = unhex(cm);
      std::vector<uint64_t> cidx(n), idx(n);
      std::vector<uint8_t> cells(2048 * n), proofs(48 * n);
      for (size_t k = 0; k < n; k++) {
        std::string c, p;
        std::cin >> cidx[k] >> idx[k] >> c >> p;
        const std::vector<uint8_t> cb = unhex(c), pb = unhex(p);
        memcpy(&cells[2048 * k], cb.data(), 2048);
        memcpy(&proofs[48 * k], pb.data(), 48);
      }
      uint64_t r[4];
      kzg::cell_batch_challenge(r, commitments.data(), u, cidx.data(), idx.data(), cells.data(), proofs.data(), n);
      uint8_t o[32];
      kzg::limbs_to_be32(o, r);
      std::cout << hex(o, 32) << "\n";
    } else {
      std::cout << "unknown\n";
    }
    std::cout.flush();
  }
  return 0;
}
