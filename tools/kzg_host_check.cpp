// Host pieces of the EIP-4844 proof entries (constantine_b200/csrc/eth_kzg_host.hpp) behind a line protocol, so that the CPU suite can
// compare them with hashlib and the exact tier (tests/test_kzg_proof_host.py builds this with the host compiler):
//   sha <hex>                    -> SHA-256 digest (hex); "sha -" hashes the empty string
//   challenge <blob> <commit>    -> the Fiat-Shamir challenge of compute_blob_kzg_proof, 32 bytes big-endian (hex)
//   commitment <hex48>           -> the cttEthKzg status of bytes_to_kzg_commitment
//   roots                        -> the 4096 brp roots of unity, canonical, 32 bytes big-endian (hex), one per line
//   blinding <bytes32> <n> <z_1> .. <z_n>  -> the r of verify_blob_kzg_proof_batch for those caller bytes and opening challenges (each
//                                   32 bytes big-endian, canonical): "<1 if the caller's bytes were used, else 0> <r, 32 bytes big-endian>"
#include <cstdio>
#include <iostream>
#include <string>
#include <vector>
#include "eth_kzg_host.hpp"

using namespace b200::kzg;

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

int main() {
  std::string cmd;
  while (std::cin >> cmd) {
    if (cmd == "sha") {
      std::string a; std::cin >> a;
      const std::vector<uint8_t> m = unhex(a);
      uint8_t out[32];
      sha256(out, m.data(), m.size());
      std::cout << hex(out, 32) << "\n";
    } else if (cmd == "challenge") {
      std::string a, b; std::cin >> a >> b;
      const std::vector<uint8_t> blob = unhex(a), cm = unhex(b);
      if (blob.size() != BYTES_PER_BLOB || cm.size() != 48) { std::cout << "bad-length\n"; continue; }
      uint64_t z[4];
      fiat_shamir_challenge(z, blob.data(), cm.data());
      uint8_t out[32];
      limbs_to_be32(out, z);
      std::cout << hex(out, 32) << "\n";
    } else if (cmd == "commitment") {
      std::string a; std::cin >> a;
      const std::vector<uint8_t> cm = unhex(a);
      std::cout << (cm.size() == 48 ? check_commitment(cm.data()) : -1) << "\n";
    } else if (cmd == "roots") {
      const std::vector<Fr> roots = brp_roots_of_unity();
      for (const Fr& r : roots) {
        uint64_t c[4];
        fr_from_mont(c, r);
        uint8_t out[32];
        limbs_to_be32(out, c);
        std::cout << hex(out, 32) << "\n";
      }
    } else if (cmd == "blinding") {
      std::string rb;
      size_t n = 0;
      std::cin >> rb >> n;
      const std::vector<uint8_t> rnd = unhex(rb);
      std::vector<Fr> zm(n);
      for (size_t i = 0; i < n; i++) {
        std::string a; std::cin >> a;
        uint64_t z[4];
        be32_to_limbs(z, unhex(a).data());
        zm[i] = fr_to_mont(z);
      }
      uint64_t r[4];
      const bool caller = blob_batch_blinding(r, rnd.data(), zm.data(), n);
      uint8_t out[32];
      limbs_to_be32(out, r);
      std::cout << (caller ? 1 : 0) << " " << hex(out, 32) << "\n";
    } else {
      std::cout << "unknown\n";
    }
    std::cout.flush();
  }
  return 0;
}
