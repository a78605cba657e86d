// The host part of hashing Ethereum BLS messages to G2, shared by verification (eth_bls.cu, which defines these) and signing
// (eth_bls_sign.cu): expand_message_xmd runs on the host, the rest of hash to G2 on the device (h2c_kernels.cuh).
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

namespace b200 {
namespace ethbls {

struct Span { const uint8_t* data; size_t len; };   // ctt_span
constexpr size_t UNIFORM_BYTES = 256;

// RFC 9380 section 5.3.1 with SHA-256 and len_in_bytes = 256 (ell = 8)
void expand_message_xmd(uint8_t out[UNIFORM_BYTES], const uint8_t* msg, size_t msg_len, const uint8_t* dst, size_t dst_len);
// uniform = n x 256 bytes, expand_message_xmd of each message under BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_, on host threads
void expand_all(std::vector<uint8_t>& uniform, const Span* messages, size_t n);

}  // namespace ethbls
}  // namespace b200
