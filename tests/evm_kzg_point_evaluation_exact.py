"""Exact tier of the EIP-4844 POINT_EVALUATION precompile (test infrastructure): Python integers and hashlib, no code shared with the
product.

reference constantine/ethereum_evm_precompiles.nim:1245-1297 (eth_evm_kzg_point_evaluation). The input is 192 bytes,
versioned_hash(32) | z(32) | y(32) | commitment(48) | proof(48). Checks in order: the input length (192), the output length (64), the
versioned hash 0x01 || sha256(commitment)[1:], then verify_kzg_proof (kzg_verify_exact.status_kzg_proof for the input checks; the
pairing decides the rest). On success the output is FIELD_ELEMENTS_PER_BLOB || r, 32 big-endian bytes each.
"""
import hashlib

import kzg_exact as K

RECORD_BYTES, OUT_BYTES = 192, 64
SUCCESS, INVALID_INPUT_SIZE, INVALID_OUTPUT_SIZE, VERIFICATION_FAILURE = (
    "cttEVM_Success", "cttEVM_InvalidInputSize", "cttEVM_InvalidOutputSize", "cttEVM_VerificationFailure")
OUTPUT = K.N.to_bytes(32, "big") + K.R.to_bytes(32, "big")


def versioned_hash(commitment: bytes) -> bytes:
    """kzg_to_versioned_hash: 0x01 || sha256(commitment)[1:]."""
    return b"\x01" + hashlib.sha256(commitment).digest()[1:]


def record(commitment: bytes, z: bytes, y: bytes, proof: bytes, vh: bytes = None) -> bytes:
    """The precompile's input for one opening; vh defaults to the commitment's versioned hash."""
    return (versioned_hash(commitment) if vh is None else vh) + z + y + commitment + proof


def split(inputs: bytes):
    """(versioned_hash, z, y, commitment, proof) of a 192-byte input."""
    return inputs[:32], inputs[32:64], inputs[64:96], inputs[96:144], inputs[144:192]


def status(inputs: bytes, out_len: int, kzg_status) -> str:
    """The precompile's status; kzg_status(commitment, z, y, proof) is verify_kzg_proof's (0 when the opening verifies)."""
    if len(inputs) != RECORD_BYTES:
        return INVALID_INPUT_SIZE
    if out_len != OUT_BYTES:
        return INVALID_OUTPUT_SIZE
    vh, z, y, c, p = split(inputs)
    if versioned_hash(c) != vh:
        return VERIFICATION_FAILURE
    return SUCCESS if kzg_status(c, z, y, p) == 0 else VERIFICATION_FAILURE
