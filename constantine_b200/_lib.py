"""ctypes loader for libctt_b200_msm.so (the C-ABI shared library built from constantine_b200/csrc/).

There is no Python or CPU fallback: if the library is missing, loading raises; if no CUDA device is present,
the first compute call aborts inside the library with a message on stderr.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CTT_B200_LIB", os.path.join(_HERE, "lib", "libctt_b200_msm.so"))   # override: experiments with variant builds
_lib = None


class Stats(ctypes.Structure):
    _fields_ = [("c", ctypes.c_int), ("num_windows", ctypes.c_int),
                ("entries", ctypes.c_ulonglong), ("total_buckets", ctypes.c_ulonglong),
                ("kernel_launches", ctypes.c_int),
                ("ms_h2d", ctypes.c_float), ("ms_digits", ctypes.c_float), ("ms_sort", ctypes.c_float),
                ("ms_accumulate", ctypes.c_float), ("ms_fixup", ctypes.c_float), ("ms_reduce", ctypes.c_float),
                ("ms_d2h_tail", ctypes.c_float), ("ms_total", ctypes.c_float),
                ("groups", ctypes.c_int), ("slice_len", ctypes.c_int), ("affine_levels", ctypes.c_int),
                ("ms_affine", ctypes.c_float)]


def load():
    """Load the shared library (once). Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). constantine_b200 has no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.ctt_b200_msm_device.argtypes = [ci, ci, vp, vp, vp, sz, ci, ci, ci, ci]
    lib.ctt_b200_msm_device.restype = ci
    lib.ctt_b200_msm_device_digits.argtypes = [ci, vp, vp, vp, sz, ci, ci, ci, ci]
    lib.ctt_b200_msm_device_digits.restype = ci
    lib.ctt_b200_combine_window_digits.argtypes = [ci, ci, vp, vp, ci, ci]
    lib.ctt_b200_combine_window_digits.restype = ci
    lib.ctt_b200_msm_host.argtypes = [ci, ci, vp, vp, vp, sz, ci]
    lib.ctt_b200_msm_host.restype = ci
    lib.ctt_b200_sum_partials.argtypes = [ci, ci, vp, vp, sz]
    lib.ctt_b200_sum_partials.restype = ci
    lib.ctt_b200_plan.argtypes = [ci, sz, ci, ctypes.POINTER(ci), ctypes.POINTER(ci)]
    lib.ctt_b200_plan.restype = ci
    lib.ctt_b200_bases_upload.argtypes = [ci, vp, sz]
    lib.ctt_b200_bases_upload.restype = vp
    lib.ctt_b200_bases_free.argtypes = [vp]
    lib.ctt_b200_bases_free.restype = None
    lib.ctt_b200_bases_precompute.argtypes = [vp, ci]
    lib.ctt_b200_bases_precompute.restype = ci
    lib.ctt_b200_msm_cached_bases.argtypes = [vp, ci, vp, vp, sz, ci]
    lib.ctt_b200_msm_cached_bases.restype = ci
    lib.ctt_b200_msm_batch_host.argtypes = [ci, ci, vp, vp, vp, sz, sz, ci, ci]
    lib.ctt_b200_msm_batch_host.restype = ci
    lib.ctt_b200_msm_batch_cached_bases.argtypes = [vp, ci, vp, vp, sz, sz, ci, ci]
    lib.ctt_b200_msm_batch_cached_bases.restype = ci
    lib.ctt_b200_bases_precompute_for.argtypes = [vp, sz, ci]
    lib.ctt_b200_bases_precompute_for.restype = ci
    lib.ctt_b200_sum_reduce_host.argtypes = [ci, ci, vp, vp, sz]
    lib.ctt_b200_sum_reduce_host.restype = ci
    lib.ctt_b200_last_stats.argtypes = [ctypes.POINTER(Stats)]
    lib.ctt_b200_last_stats.restype = None
    lib.ctt_b200_set_tuning.argtypes = [ci, ci, ci]
    lib.ctt_b200_set_tuning.restype = None
    lib.ctt_b200_set_concurrency.argtypes = [ci]
    lib.ctt_b200_set_concurrency.restype = None
    lib.ctt_b200_set_groups.argtypes = [ci]
    lib.ctt_b200_set_groups.restype = None
    lib.ctt_b200_set_affine_levels.argtypes = [ci]
    lib.ctt_b200_set_affine_levels.restype = None
    lib.ctt_b200_set_reduce_mode.argtypes = [ci]
    lib.ctt_b200_set_reduce_mode.restype = None
    lib.ctt_b200_set_input_chunks.argtypes = [ci]
    lib.ctt_b200_set_input_chunks.restype = None
    lib.ctt_b200_set_point_chunks.argtypes = [ci]
    lib.ctt_b200_set_point_chunks.restype = None
    lib.ctt_b200_set_stream.argtypes = [vp]
    lib.ctt_b200_set_stream.restype = None
    lib.ctt_b200_sm_count.argtypes = []
    lib.ctt_b200_sm_count.restype = ci
    lib.ctt_b200_set_devices.argtypes = [ctypes.POINTER(ci), ci]
    lib.ctt_b200_set_devices.restype = ci
    lib.ctt_b200_device_count.argtypes = []
    lib.ctt_b200_device_count.restype = ci
    lib.ctt_b200_test_field_op.argtypes = [ci, ci, vp, vp, vp, sz]
    lib.ctt_b200_test_field_op.restype = ci
    lib.ctt_b200_test_ct_op.argtypes = [ci, ci, vp, vp, vp, sz]
    lib.ctt_b200_test_ct_op.restype = ci
    lib.ctt_b200_test_ec_op.argtypes = [ci, ci, vp, vp, vp, sz]
    lib.ctt_b200_test_ec_op.restype = ci
    if hasattr(lib, "ctt_b200_scalar_mul_u64"):
        lib.ctt_b200_scalar_mul_u64.argtypes = [ci, vp, vp, sz, vp]
        lib.ctt_b200_scalar_mul_u64.restype = ci
    for nm in ("ctt_eth_evm_bls12381_g1msm", "ctt_eth_evm_bls12381_g2msm"):
        fn = getattr(lib, nm)
        fn.argtypes = [vp, sz, vp, sz]
        fn.restype = ctypes.c_ubyte
    lib.ctt_eth_evm_bn254_ecpairingcheck.argtypes = [vp, sz, vp, sz]
    lib.ctt_eth_evm_bn254_ecpairingcheck.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_evm_bn254_ecpairingcheck_batch.argtypes = [vp, vp, vp, sz, vp, sz]
    lib.ctt_b200_eth_evm_bn254_ecpairingcheck_batch.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_evm_bn254_last_timing.argtypes = [ctypes.POINTER(ctypes.c_float)] * 4
    lib.ctt_b200_eth_evm_bn254_last_timing.restype = None
    for nm in ("ctt_eth_evm_bls12381_pairingcheck", "ctt_eth_evm_bls12381_map_fp_to_g1", "ctt_eth_evm_bls12381_map_fp2_to_g2"):
        fn = getattr(lib, nm)
        fn.argtypes = [vp, sz, vp, sz]
        fn.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_evm_bls12381_pairingcheck_batch.argtypes = [vp, vp, vp, sz, vp, sz]
    lib.ctt_b200_eth_evm_bls12381_pairingcheck_batch.restype = ctypes.c_ubyte
    for nm in ("ctt_b200_eth_evm_bls12381_map_fp_to_g1_batch", "ctt_b200_eth_evm_bls12381_map_fp2_to_g2_batch"):
        fn = getattr(lib, nm)
        fn.argtypes = [vp, vp, vp, sz]
        fn.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_evm_bls12381_last_timing.argtypes = [ctypes.POINTER(ctypes.c_float)] * 5
    lib.ctt_b200_eth_evm_bls12381_last_timing.restype = None
    for nm in ("bn254_g1add", "bn254_g1mul", "bls12381_g1add", "bls12381_g2add", "bls12381_g1mul", "bls12381_g2mul"):
        fn = getattr(lib, "ctt_eth_evm_" + nm)
        fn.argtypes = [vp, sz, vp, sz]
        fn.restype = ctypes.c_ubyte
        fn = getattr(lib, "ctt_b200_eth_evm_" + nm + "_batch")
        fn.argtypes = [vp, vp, vp, sz]
        fn.restype = ctypes.c_ubyte
    lib.ctt_eth_evm_ecrecover.argtypes = [vp, sz, vp, sz]
    lib.ctt_eth_evm_ecrecover.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_evm_ecrecover_batch.argtypes = [vp, vp, vp, sz]
    lib.ctt_b200_eth_evm_ecrecover_batch.restype = ctypes.c_ubyte
    for nm in ("sha256", "ripemd160", "modexp"):
        fn = getattr(lib, "ctt_eth_evm_" + nm)
        fn.argtypes = [vp, sz, vp, sz]
        fn.restype = ctypes.c_ubyte
    lib.ctt_eth_evm_modexp_result_size.argtypes = [ctypes.POINTER(ctypes.c_uint64), vp, sz]
    lib.ctt_eth_evm_modexp_result_size.restype = ctypes.c_ubyte
    for nm in ("sha256", "ripemd160"):
        fn = getattr(lib, "ctt_b200_eth_evm_" + nm + "_batch")
        fn.argtypes = [vp, vp, sz, vp, sz]
        fn.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_evm_modexp_batch.argtypes = [vp, vp, vp, vp, sz, vp, sz]
    lib.ctt_b200_eth_evm_modexp_batch.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_evm_ecops_last_timing.argtypes = [ctypes.POINTER(ctypes.c_float)]
    lib.ctt_b200_eth_evm_ecops_last_timing.restype = None
    for nm, args in (("sign", [vp, vp, vp, sz, ci]), ("verify", [vp, vp, sz, vp]), ("recover_pubkey", [vp, vp, sz, vp, ci]),
                     ("recover_pubkey_from_digest", [vp, vp, vp, ci]), ("derive_pubkey", [vp, vp]),
                     ("sign_batch", [vp, vp, vp, vp, sz, vp, sz, ci]), ("verify_batch", [vp, vp, vp, vp, sz, vp, sz]),
                     ("recover_pubkey_batch", [vp, vp, vp, vp, vp, sz, vp, sz]),
                     ("recover_pubkey_from_digest_batch", [vp, vp, vp, vp, vp, sz]), ("derive_pubkey_batch", [vp, vp, vp, sz])):
        fn = getattr(lib, "ctt_b200_eth_ecdsa_" + nm)
        fn.argtypes = args
        fn.restype = ci
    lib.ctt_b200_eth_ecdsa_last_timing.argtypes = [ctypes.POINTER(ctypes.c_float)] * 2
    lib.ctt_b200_eth_ecdsa_last_timing.restype = None
    lib.ctt_b200_test_bn254_pairing.argtypes = [vp, vp, sz, vp]
    lib.ctt_b200_test_bn254_pairing.restype = ci
    lib.ctt_b200_eth_kzg_context_new.argtypes = [vp]
    lib.ctt_b200_eth_kzg_context_new.restype = vp
    lib.ctt_b200_eth_kzg_context_new_compressed.argtypes = [vp, ctypes.POINTER(ci)]
    lib.ctt_b200_eth_kzg_context_new_compressed.restype = vp
    lib.ctt_b200_eth_kzg_context_precompute.argtypes = [vp, ci]
    lib.ctt_b200_eth_kzg_context_precompute.restype = ci
    lib.ctt_b200_eth_kzg_context_delete.argtypes = [vp]
    lib.ctt_b200_eth_kzg_context_delete.restype = None
    lib.ctt_b200_eth_kzg_blob_to_kzg_commitment.argtypes = [vp, vp, vp]
    lib.ctt_b200_eth_kzg_blob_to_kzg_commitment.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_compute_kzg_proof.argtypes = [vp, vp, vp, vp, vp]
    lib.ctt_b200_eth_kzg_compute_kzg_proof.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_compute_blob_kzg_proof.argtypes = [vp, vp, vp, vp]
    lib.ctt_b200_eth_kzg_compute_blob_kzg_proof.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_blobs_to_kzg_commitments.argtypes = [vp, vp, vp, sz, ctypes.POINTER(sz)]
    lib.ctt_b200_eth_kzg_blobs_to_kzg_commitments.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_compute_blob_kzg_proofs.argtypes = [vp, vp, vp, vp, sz, ctypes.POINTER(sz)]
    lib.ctt_b200_eth_kzg_compute_blob_kzg_proofs.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_last_timing.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float)]
    lib.ctt_b200_eth_kzg_last_timing.restype = None
    lib.ctt_b200_eth_kzg_context_load_peerdas.argtypes = [vp, vp]
    lib.ctt_b200_eth_kzg_context_load_peerdas.restype = ci
    lib.ctt_b200_eth_kzg_compute_cells.argtypes = [vp, vp, vp]
    lib.ctt_b200_eth_kzg_compute_cells.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_compute_cells_and_kzg_proofs.argtypes = [vp, vp, vp, vp]
    lib.ctt_b200_eth_kzg_compute_cells_and_kzg_proofs.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_compute_cells_and_kzg_proofs_batch.argtypes = [vp, vp, vp, vp, sz, ctypes.POINTER(sz)]
    lib.ctt_b200_eth_kzg_compute_cells_and_kzg_proofs_batch.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_last_das_timing.argtypes = [ctypes.POINTER(ctypes.c_float)] * 4
    lib.ctt_b200_eth_kzg_last_das_timing.restype = None
    lib.ctt_b200_eth_kzg_recover_cells_and_kzg_proofs.argtypes = [vp, vp, vp, vp, vp, sz]
    lib.ctt_b200_eth_kzg_recover_cells_and_kzg_proofs.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_recover_cells_and_kzg_proofs_batch.argtypes = [vp, vp, vp, vp, vp, vp, sz, ctypes.POINTER(sz)]
    lib.ctt_b200_eth_kzg_recover_cells_and_kzg_proofs_batch.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_context_load_g2_setup.argtypes = [vp, vp]
    lib.ctt_b200_eth_kzg_context_load_g2_setup.restype = ci
    lib.ctt_b200_eth_kzg_verify_cell_kzg_proof_batch.argtypes = [vp, vp, vp, vp, vp, sz, vp]
    lib.ctt_b200_eth_kzg_verify_cell_kzg_proof_batch.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_verify_kzg_proof.argtypes = [vp, vp, vp, vp, vp]
    lib.ctt_b200_eth_kzg_verify_kzg_proof.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_verify_blob_kzg_proof.argtypes = [vp, vp, vp, vp]
    lib.ctt_b200_eth_kzg_verify_blob_kzg_proof.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_verify_blob_kzg_proof_batch.argtypes = [vp, vp, vp, vp, sz, vp]
    lib.ctt_b200_eth_kzg_verify_blob_kzg_proof_batch.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_last_verify_timing.argtypes = [ctypes.POINTER(ctypes.c_float)] * 5
    lib.ctt_b200_eth_kzg_last_verify_timing.restype = None
    lib.ctt_b200_eth_kzg_verify_kzg_proofs.argtypes = [vp, vp, vp, vp, vp, vp, sz]
    lib.ctt_b200_eth_kzg_verify_kzg_proofs.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_evm_kzg_point_evaluation.argtypes = [vp, vp, sz, vp, sz]
    lib.ctt_b200_eth_evm_kzg_point_evaluation.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_evm_kzg_point_evaluation_batch.argtypes = [vp, vp, vp, vp, sz]
    lib.ctt_b200_eth_evm_kzg_point_evaluation_batch.restype = ctypes.c_ubyte
    lib.ctt_b200_eth_kzg_last_point_eval_timing.argtypes = [ctypes.POINTER(ctypes.c_float)] * 4
    lib.ctt_b200_eth_kzg_last_point_eval_timing.restype = None
    ub = ctypes.c_uint8
    lib.ctt_eth_bls_batch_verify.argtypes = [vp, vp, vp, sz, vp]
    lib.ctt_eth_bls_batch_verify.restype = ub
    lib.ctt_eth_bls_batch_verify_parallel.argtypes = [vp, vp, vp, vp, sz, vp]
    lib.ctt_eth_bls_batch_verify_parallel.restype = ub
    lib.ctt_eth_bls_aggregate_verify.argtypes = [vp, vp, sz, vp]
    lib.ctt_eth_bls_aggregate_verify.restype = ub
    lib.ctt_b200_eth_bls_deserialize_pubkey_compressed.argtypes = [vp, vp]
    lib.ctt_b200_eth_bls_deserialize_pubkey_compressed.restype = ci
    lib.ctt_b200_eth_bls_deserialize_signature_compressed.argtypes = [vp, vp]
    lib.ctt_b200_eth_bls_deserialize_signature_compressed.restype = ci
    lib.ctt_b200_eth_bls_last_timing.argtypes = [ctypes.POINTER(ctypes.c_float)] * 6
    lib.ctt_b200_eth_bls_last_timing.restype = None
    lib.ctt_b200_eth_bls_batch_verify_sets.argtypes = [vp, vp, vp, vp, vp, sz, vp, ctypes.POINTER(sz)]
    lib.ctt_b200_eth_bls_batch_verify_sets.restype = ub
    lib.ctt_b200_eth_bls_verify_sets.argtypes = [vp, vp, vp, vp, vp, sz, vp]
    lib.ctt_b200_eth_bls_verify_sets.restype = ub
    lib.ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch.argtypes = [vp, vp, vp, sz]
    lib.ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch.restype = ci
    lib.ctt_b200_eth_bls_deserialize_signatures_compressed_batch.argtypes = [vp, vp, vp, sz]
    lib.ctt_b200_eth_bls_deserialize_signatures_compressed_batch.restype = ci
    lib.ctt_b200_eth_bls_registry_from_compressed.argtypes = [vp, sz, vp, ctypes.POINTER(sz), ctypes.POINTER(ci)]
    lib.ctt_b200_eth_bls_registry_from_compressed.restype = vp
    for nm, args in (("sign", [vp, vp, vp, sz]), ("sign_batch", [vp, vp, vp, vp, sz, vp, sz]), ("derive_pubkey", [vp, vp]),
                     ("derive_pubkey_batch", [vp, vp, vp, sz]), ("serialize_pubkey_compressed", [vp, vp]),
                     ("serialize_signature_compressed", [vp, vp]), ("serialize_pubkeys_compressed_batch", [vp, vp, sz]),
                     ("serialize_signatures_compressed_batch", [vp, vp, sz])):
        fn = getattr(lib, "ctt_b200_eth_bls_" + nm)
        fn.argtypes = args
        fn.restype = ci
    lib.ctt_b200_eth_bls_signer_last_timing.argtypes = [ctypes.POINTER(ctypes.c_float)] * 3
    lib.ctt_b200_eth_bls_signer_last_timing.restype = None
    u32 = ctypes.c_uint32
    for nm, args in (("derive_master_secret_key", [vp, vp, sz]), ("derive_master_secret_keys_batch", [vp, vp, vp, sz, vp, sz]),
                     ("derive_child_secret_key", [vp, vp, u32]), ("derive_child_secret_keys_batch", [vp, vp, vp, vp, sz]),
                     ("derive_path_batch", [vp, vp, vp, vp, sz, vp, sz, vp, vp, sz, sz])):
        fn = getattr(lib, "ctt_b200_eth_eip2333_" + nm)
        fn.argtypes = args
        fn.restype = ci
    lib.ctt_b200_eth_eip2333_last_stats.argtypes = [ctypes.POINTER(ctypes.c_float)] * 2 + [ctypes.POINTER(ctypes.c_uint64)] * 2
    lib.ctt_b200_eth_eip2333_last_stats.restype = None
    lib.ctt_b200_fft_domain_new.argtypes = [ci, vp, ci, ctypes.POINTER(ci)]
    lib.ctt_b200_fft_domain_new.restype = vp
    lib.ctt_b200_fft_domain_free.argtypes = [vp]
    lib.ctt_b200_fft_domain_free.restype = None
    lib.ctt_b200_fft.argtypes = [vp, ci, vp, vp, sz, sz, vp]
    lib.ctt_b200_fft.restype = ci
    lib.ctt_b200_fft_device.argtypes = [vp, ci, vp, vp, sz, sz, vp]
    lib.ctt_b200_fft_device.restype = ci
    lib.ctt_b200_fft_last_timing.argtypes = [ctypes.POINTER(ctypes.c_float)] * 3
    lib.ctt_b200_fft_last_timing.restype = None
    lib.ctt_b200_test_hash_to_g2.argtypes = [vp, sz, vp, sz, vp]
    lib.ctt_b200_test_hash_to_g2.restype = ci
    lib.ctt_b200_test_map_to_g2.argtypes = [vp, sz, vp]
    lib.ctt_b200_test_map_to_g2.restype = ci
    lib.ctt_b200_test_pairing.argtypes = [vp, vp, sz, vp]
    lib.ctt_b200_test_pairing.restype = ci
    lib.ctt_threadpool_new.argtypes = [ci]
    lib.ctt_threadpool_new.restype = vp
    lib.ctt_threadpool_shutdown.argtypes = [vp]
    lib.ctt_threadpool_shutdown.restype = None
    lib.ctt_cpu_get_num_threads_os.argtypes = []
    lib.ctt_cpu_get_num_threads_os.restype = ci
    _lib = lib
    return lib


def named_msm(symbol: str):
    """Return the named reference-ABI export, e.g. ctt_bls12_381_g1_jac_multi_scalar_mul_big_coefs_vartime_parallel."""
    lib = load()
    fn = getattr(lib, symbol)
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    fn.argtypes = [vp, vp, vp, vp, sz] if symbol.endswith("_parallel") else [vp, vp, vp, sz]
    fn.restype = None
    return fn
