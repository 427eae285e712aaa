"""ctypes binding of include/b200snark.h (one-to-one; see the header for semantics and the reference
interfaces each entry point replaces)."""
import ctypes
import os
import secrets
from ctypes import POINTER, c_char_p, c_int32, c_uint32, c_uint64, c_void_p

import numpy as np

BLS12_381, BN254, BLS12_377 = 0, 1, 2
MEM_HOST, MEM_DEVICE = 0, 1
QAP_LIBSNARK, QAP_CIRCOM = 0, 1   # QAP reduction of a Groth16 key: ark-groth16's LibsnarkReduction / ark-circom's CircomReduction

_HERE = os.path.dirname(os.path.abspath(__file__))


def lib_path():
    return os.path.join(_HERE, "libb200snark.so")


class B2SError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200snark error {code}: {msg}")
        self.code = code


class PkDesc(ctypes.Structure):
    _fields_ = [
        ("n_instance", c_uint64), ("n_witness", c_uint64), ("domain_size", c_uint64),
        ("alpha_g1", c_void_p), ("beta_g1", c_void_p), ("delta_g1", c_void_p),
        ("beta_g2", c_void_p), ("delta_g2", c_void_p),
        ("a_query", c_void_p), ("a_off", c_uint64), ("a_len", c_uint64),
        ("b_g1_query", c_void_p), ("b1_off", c_uint64), ("b1_len", c_uint64),
        ("b_g2_query", c_void_p), ("b2_off", c_uint64), ("b2_len", c_uint64),
        ("h_query", c_void_p), ("h_off", c_uint64), ("h_len", c_uint64),
        ("l_query", c_void_p), ("l_off", c_uint64), ("l_len", c_uint64),
    ]


GR1CS_MAX_ARITY = 8
NOT_FOUND = np.uint64(0xFFFFFFFFFFFFFFFF)   # first_unsat of a satisfied predicate
# instance outlining strategies (b2s_outline): ark-relations' outline_r1cs / outline_sr1cs
OUTLINE_R1CS, OUTLINE_SR1CS = 1, 2
# scalar-field moduli, for the Montgomery form of the Python-int coefficients gr1cs_upload takes
FR_MODULUS = {BLS12_381: 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001,
              BN254: 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001,
              BLS12_377: 0x12AB655E9A2CA55660B44D1E5C37B00159AA76FED00000010A11800000000001}


class ZkeyInfo(ctypes.Structure):
    _fields_ = [("n_vars", c_uint64), ("n_public", c_uint64), ("domain_size", c_uint64), ("n_coeffs", c_uint64)]


class R1csFileInfo(ctypes.Structure):
    _fields_ = [(n, c_uint64) for n in ("n_wires", "n_pub_out", "n_pub_in", "n_prv_in", "n_labels", "n_constraints", "domain_size")]


class PredicateDesc(ctypes.Structure):
    _fields_ = [
        ("arity", c_uint32), ("n_terms", c_uint32),
        ("term_coeffs", c_void_p), ("term_offsets", c_void_p), ("factor_var", c_void_p), ("factor_pow", c_void_p),
        ("n_rows", c_uint64),
        ("row_ptr", c_void_p * GR1CS_MAX_ARITY), ("col", c_void_p * GR1CS_MAX_ARITY), ("coeff", c_void_p * GR1CS_MAX_ARITY),
    ]


class Gr1csPredInfo(ctypes.Structure):
    _fields_ = [("arity", c_uint32), ("reserved", c_uint32), ("n_rows", c_uint64), ("nnz", c_uint64 * GR1CS_MAX_ARITY)]


class PredicateLcmapDesc(ctypes.Structure):
    _fields_ = [
        ("arity", c_uint32), ("n_terms", c_uint32),
        ("term_coeffs", c_void_p), ("term_offsets", c_void_p), ("factor_var", c_void_p), ("factor_pow", c_void_p),
        ("n_rows", c_uint64),
        ("args", c_void_p * GR1CS_MAX_ARITY),
    ]


class Outline(ctypes.Structure):
    """b2s_outline: the strategy (OUTLINE_R1CS / OUTLINE_SR1CS) and the upload index of the predicate that gets the tie rows"""
    _fields_ = [("strategy", c_int32), ("pred", c_uint32)]


def _mont_limbs(r, xs):
    """Python ints -> uint32[len(xs) * 8] Montgomery limbs mod r"""
    out = np.zeros((len(xs), 8), dtype=np.uint32)
    for i, x in enumerate(xs):
        v = (x % r) * (1 << 256) % r
        out[i] = [(v >> (32 * j)) & 0xFFFFFFFF for j in range(8)]
    return out.reshape(-1)


def _set_poly(d, r, terms, keep):
    """the polynomial fields of a predicate descriptor from terms [(coeff, [(argument, exponent), ...])]; the arrays go to keep"""
    offs = np.zeros(len(terms) + 1, dtype=np.uint32)
    offs[1:] = np.cumsum([len(mono) for _, mono in terms])
    arrs = [_mont_limbs(r, [c for c, _ in terms]), offs, np.array([v for _, mono in terms for v, _ in mono], dtype=np.uint32),
            np.array([e for _, mono in terms for _, e in mono], dtype=np.uint32)]
    keep += arrs
    d.term_coeffs, d.term_offsets, d.factor_var, d.factor_pow = (a.ctypes.data for a in arrs)


def _csr(r, matrix):
    """Matrix (rows of (coeff, col), as to_matrices() returns it) -> (row_ptr u64, col u32, coeff Montgomery limbs)"""
    row_ptr = np.zeros(len(matrix) + 1, dtype=np.uint64)
    row_ptr[1:] = np.cumsum([len(row) for row in matrix], dtype=np.uint64)
    cols = np.array([col for row in matrix for _, col in row], dtype=np.uint32)
    return row_ptr, cols, _mont_limbs(r, [c for row in matrix for c, _ in row])


class Gr1cs:
    """A device-resident GR1CS (b2s_gr1cs), the labels of its predicates in upload (BTreeMap) order and the number of
    variables (n_instance + n_witness) every assignment holds."""

    def __init__(self, handle, labels, n_vars, src_vars=None):
        self.h = handle
        self.labels = labels
        self.n_vars = n_vars
        self.src_vars = src_vars   # the source's n_instance + n_witness, for a handle from r1cs_to_sr1cs


# name -> (restype, argtypes): every symbol include/b200snark.h declares
SIGNATURES = {
    "b2s_version": (c_char_p, []),
    "b2s_ctx_create": (c_int32, [c_int32, c_int32, POINTER(c_void_p)]),
    "b2s_ctx_destroy": (None, [c_void_p]),
    "b2s_last_error": (c_char_p, [c_void_p]),
    "b2s_sizes": (c_int32, [c_void_p, POINTER(c_uint32)]),
    "b2s_launch_count": (c_uint64, [c_void_p]),
    "b2s_sync": (c_int32, [c_void_p]),
    "b2s_stream": (c_void_p, [c_void_p]),
    "b2s_ntt": (c_int32, [c_void_p, c_void_p, c_uint32, c_int32, c_int32, c_int32]),
    "b2s_msm_g1": (c_int32, [c_void_p, c_void_p, c_void_p, c_uint64, c_int32, c_int32, c_void_p]),
    "b2s_msm_g2": (c_int32, [c_void_p, c_void_p, c_void_p, c_uint64, c_int32, c_int32, c_void_p]),
    "b2s_msm_g1_partial": (c_int32, [c_void_p, c_void_p, c_void_p, c_uint64, c_int32, c_int32, c_void_p]),
    "b2s_msm_g2_partial": (c_int32, [c_void_p, c_void_p, c_void_p, c_uint64, c_int32, c_int32, c_void_p]),
    "b2s_g1_sum": (c_int32, [c_void_p, c_void_p, c_uint32, c_void_p]),
    "b2s_g2_sum": (c_int32, [c_void_p, c_void_p, c_uint32, c_void_p]),
    "b2s_r1cs_upload": (c_int32, [c_void_p, c_uint64, c_uint64, c_uint64, POINTER(c_void_p), POINTER(c_void_p),
                                  POINTER(c_void_p), POINTER(c_void_p)]),
    "b2s_r1cs_upload_lcmap": (c_int32, [c_void_p, c_uint64, c_uint64, c_uint64, POINTER(c_void_p), c_uint64, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_uint32, POINTER(c_void_p)]),
    "b2s_r1cs_free": (None, [c_void_p, c_void_p]),
    "b2s_spmv": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p]),
    "b2s_witness_map": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_void_p]),
    "b2s_witness_map_qap": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p]),
    "b2s_r1cs_domain_size": (c_uint64, [c_void_p]),
    "b2s_witness_map_sim": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_uint32, c_void_p]),
    "b2s_gr1cs_upload": (c_int32, [c_void_p, c_uint64, c_uint64, c_uint32, c_void_p, POINTER(c_void_p)]),
    "b2s_gr1cs_upload_lcmap": (c_int32, [c_void_p, c_uint64, c_uint64, c_uint32, c_void_p, c_uint64, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_uint32, POINTER(c_void_p)]),
    "b2s_gr1cs_free": (None, [c_void_p, c_void_p]),
    "b2s_gr1cs_check": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_int32, c_void_p, c_void_p]),
    "b2s_r1cs_check": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_int32, c_void_p, c_void_p]),
    "b2s_r1cs_to_sr1cs": (c_int32, [c_void_p, c_void_p, POINTER(c_void_p)]),
    "b2s_sr1cs_assignment": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_int32, c_void_p]),
    "b2s_gr1cs_info": (c_int32, [c_void_p, c_void_p, POINTER(c_uint64), POINTER(c_uint32), POINTER(Gr1csPredInfo), c_uint32]),
    "b2s_gr1cs_export": (c_int32, [c_void_p, c_void_p, c_uint32, c_uint32, c_void_p, c_uint64, c_void_p, c_uint64, c_void_p, c_uint64]),
    "b2s_gr1cs_upload_lcmap_outline": (c_int32, [c_void_p, c_uint64, c_uint64, c_uint32, c_void_p, c_uint64, c_void_p, c_void_p, c_void_p,
                                                 c_void_p, c_uint32, POINTER(Outline), POINTER(c_void_p)]),
    "b2s_r1cs_upload_lcmap_outline": (c_int32, [c_void_p, c_uint64, c_uint64, c_uint64, POINTER(c_void_p), c_uint64, c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_uint32, POINTER(Outline), POINTER(c_void_p)]),
    "b2s_gr1cs_outline_assignment": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_int32, c_void_p]),
    "b2s_r1cs_outline_assignment": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_int32, c_void_p]),
    "b2s_pk_upload": (c_int32, [c_void_p, POINTER(PkDesc), c_int32, POINTER(c_void_p)]),
    "b2s_pk_upload_qap": (c_int32, [c_void_p, POINTER(PkDesc), c_int32, c_int32, POINTER(c_void_p)]),
    "b2s_pk_free": (None, [c_void_p, c_void_p]),
    "b2s_groth16_setup": (c_int32, [c_void_p, c_void_p, c_void_p, POINTER(c_void_p)] + [c_void_p] * 5),
    "b2s_groth16_setup_qap": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, POINTER(c_void_p)] + [c_void_p] * 5),
    "b2s_pk_query": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_uint64]),
    "b2s_groth16_prove": (c_int32, [c_void_p] * 10),
    "b2s_groth16_prove_shard": (c_int32, [c_void_p] * 9),
    "b2s_groth16_prove_resident": (c_int32, [c_void_p] * 9),
    "b2s_groth16_prove_shard_resident": (c_int32, [c_void_p] * 8),
    "b2s_groth16_prove_batch": (c_int32, [c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                                          c_void_p]),
    "b2s_profile_enable": (c_int32, [c_void_p, c_int32]),
    "b2s_profile_report": (c_int32, [c_void_p, c_char_p, c_uint64]),
    "b2s_groth16_finish": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p]),
    "b2s_serialize_g1_compressed": (c_int32, [c_void_p, c_void_p, c_uint32, c_void_p, c_uint64]),
    "b2s_serialize_g2_compressed": (c_int32, [c_void_p, c_void_p, c_uint32, c_void_p, c_uint64]),
    "b2s_proof_serialize_compressed": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint64]),
    "b2s_serialize_g1_uncompressed": (c_int32, [c_void_p, c_void_p, c_uint32, c_void_p, c_uint64]),
    "b2s_serialize_g2_uncompressed": (c_int32, [c_void_p, c_void_p, c_uint32, c_void_p, c_uint64]),
    "b2s_proof_serialize_uncompressed": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint64]),
    "b2s_vk_serialized_size": (c_uint64, [c_void_p, c_uint64, c_int32]),
    "b2s_vk_serialize": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint64, c_int32, c_void_p, c_uint64]),
    "b2s_pk_serialized_size": (c_uint64, [c_void_p, c_void_p, c_uint64, c_int32]),
    "b2s_pk_serialize": (c_int32, [c_void_p, c_void_p, c_void_p, c_uint64, c_int32, c_void_p, c_uint64]),
    "b2s_deserialize_g1": (c_int32, [c_void_p, c_void_p, c_uint64, c_uint64, c_int32, c_int32, c_void_p]),
    "b2s_deserialize_g2": (c_int32, [c_void_p, c_void_p, c_uint64, c_uint64, c_int32, c_int32, c_void_p]),
    "b2s_proof_deserialize": (c_int32, [c_void_p, c_void_p, c_uint64, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "b2s_vk_deserialize": (c_int32, [c_void_p, c_void_p, c_uint64, c_int32, c_int32] + [c_void_p] * 5
                           + [c_uint64, POINTER(c_uint64), POINTER(c_uint64)]),
    "b2s_pk_deserialize": (c_int32, [c_void_p, c_void_p, c_uint64, c_int32, c_int32, POINTER(c_void_p)]),
    "b2s_pk_deserialize_qap": (c_int32, [c_void_p, c_void_p, c_uint64, c_int32, c_int32, c_int32, POINTER(c_void_p)]),
    "b2s_zkey_read_info": (c_int32, [c_void_p, c_void_p, c_uint64, POINTER(ZkeyInfo)]),
    "b2s_zkey_load": (c_int32, [c_void_p, c_void_p, c_uint64, c_int32, POINTER(c_void_p), POINTER(c_void_p)] + [c_void_p] * 5 + [c_uint64]),
    "b2s_wtns_read": (c_int32, [c_void_p, c_void_p, c_uint64, c_uint64, c_int32, c_void_p]),
    "b2s_r1cs_file_read_info": (c_int32, [c_void_p, c_void_p, c_uint64, POINTER(R1csFileInfo)]),
    "b2s_r1cs_file_load": (c_int32, [c_void_p, c_void_p, c_uint64, POINTER(c_void_p)]),
    "b2s_vk_prepare": (c_int32, [c_void_p] * 6 + [c_uint64, POINTER(c_void_p)]),
    "b2s_pvk_free": (None, [c_void_p, c_void_p]),
    "b2s_groth16_verify_batch": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint64, c_void_p, c_void_p, c_void_p, c_int32,
                                           c_void_p]),
    "b2s_groth16_verify_batch_rlc": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint64, c_void_p, c_void_p, c_void_p,
                                               c_void_p, c_int32, POINTER(ctypes.c_uint8)]),
    "b2s_groth16_verify_batch_bytes": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint64, c_void_p, c_uint64, c_int32, c_int32,
                                                 c_void_p, c_void_p]),
    "b2s_groth16_verify_batch_rlc_bytes": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint64, c_void_p, c_uint64, c_int32,
                                                     c_void_p, c_int32, POINTER(ctypes.c_uint8), c_void_p]),
    "b2s_pairing": (c_int32, [c_void_p, c_void_p, c_void_p, c_uint64, c_int32, c_void_p]),
    "b2s_fixed_base_g1": (c_int32, [c_void_p, c_void_p, c_uint64, c_int32, c_int32, c_void_p]),
    "b2s_fixed_base_g2": (c_int32, [c_void_p, c_void_p, c_uint64, c_int32, c_int32, c_void_p]),
    "b2s_group_unique_id": (c_int32, [c_void_p]),
    "b2s_group_create": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, POINTER(c_void_p)]),
    "b2s_group_destroy": (None, [c_void_p]),
    "b2s_groth16_prove_group": (c_int32, [c_void_p] * 10),
    "b2s_groth16_prove_group_resident": (c_int32, [c_void_p] * 9),
    "b2s_poly_op": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_uint64, c_int32]),
    "b2s_poly_geom": (c_int32, [c_void_p, c_void_p, c_void_p, c_uint64, c_int32, c_void_p]),
    "b2s_poly_eval": (c_int32, [c_void_p, c_void_p, c_uint64, c_void_p, c_int32, c_void_p]),
    "b2s_field_op": (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_uint64]),
    "b2s_group_op": (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_uint64]),
}

_lib = None


def load_library():
    """Load libb200snark.so and type every exported symbol.  Raises if the library is missing: there is
    no Python or CPU substitute."""
    global _lib
    if _lib is None:
        path = lib_path()
        if not os.path.exists(path):
            raise B2SError(-1, f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`")
        lib = ctypes.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the header and the library disagree
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def random_rho(n):
    """n nonzero 128-bit integers from the OS CSPRNG, as n x 4 little-endian uint32 words (the rho of
    b2s_groth16_verify_batch_rlc)"""
    w = np.frombuffer(secrets.token_bytes(16 * n), dtype=np.uint32).reshape(n, 4).copy()
    zero = ~w.any(axis=1)
    while zero.any():
        w[zero] = np.frombuffer(secrets.token_bytes(16 * int(zero.sum())), dtype=np.uint32).reshape(-1, 4)
        zero = ~w.any(axis=1)
    return w.reshape(-1)


def _ptr(x):
    """Host numpy array or device torch tensor (or None / raw device address) -> (address, mem flag)."""
    if x is None:
        return None, MEM_HOST
    if isinstance(x, np.ndarray):
        assert x.flags["C_CONTIGUOUS"]
        return x.ctypes.data, MEM_HOST
    if isinstance(x, int):
        return x, MEM_DEVICE
    assert x.is_contiguous()  # torch tensor
    if x.is_cuda:
        # The library launches on its own stream (b2s_stream).  Whatever torch queued to produce this tensor must be
        # finished before that stream reads it; conversely the caller keeps the tensor alive and calls Backend.sync()
        # before torch touches anything the library wrote (device-memory calls return without synchronising).
        import torch

        torch.cuda.current_stream(x.device).synchronize()
    return x.data_ptr(), (MEM_DEVICE if x.is_cuda else MEM_HOST)


def _ptrs(*bufs, same=True):
    """_ptr of several buffers -> ([addresses], the memory kind of the first).  With `same`, asserts that the buffers other
    than None share one memory kind."""
    got = [_ptr(x) for x in bufs]
    assert not same or len({m for x, (_, m) in zip(bufs, got) if x is not None}) <= 1
    return [p for p, _ in got], got[0][1]


def _nbytes(x):
    """byte size of a numpy array or torch tensor"""
    return x.nbytes if isinstance(x, np.ndarray) else x.numel() * x.element_size()


def _draw_rho(n, mem, like):
    """random_rho(n) in `mem`: a numpy array, or an int32 tensor on the device of the tensor `like`"""
    rho = random_rho(n)
    if mem == MEM_DEVICE:
        import torch

        rho = torch.from_numpy(rho.view(np.int32)).to(like.device)
    return rho


def _zeros(shapes, dtype, mem, like):
    """Zero-filled output arrays of one shape each: numpy `dtype` (np.uint32 / np.uint64) on the host, or torch tensors of
    the signed type of the same width on the device of the tensor `like`.  torch's stream is synchronised after a device
    fill, so that the zeros are in place before the library's stream writes."""
    if mem == MEM_HOST:
        return [np.zeros(s, dtype=dtype) for s in shapes]
    import torch

    tdtype = torch.int64 if np.dtype(dtype).itemsize == 8 else torch.int32
    out = [torch.zeros(s, dtype=tdtype, device=like.device) for s in shapes]
    torch.cuda.current_stream(like.device).synchronize()
    return out


class Backend:
    """One `b2s_ctx`: a curve bound to one GPU.  Buffers are numpy uint32/uint64 arrays (host) or
    CUDA torch tensors (device), already in the C-ABI layout (Montgomery limbs)."""

    def __init__(self, curve=BLS12_381, device=0):
        self.h = None
        self._r1cs_vars = {}   # n_instance + n_witness of each matrix handle, for the width check of r1cs_check
        self._r1cs_src_vars = {}   # of an outlined matrix handle: the variables before outlining (outline_assignment's input)
        self.lib = load_library()
        h = c_void_p()
        st = self.lib.b2s_ctx_create(curve, device, ctypes.byref(h))
        if st != 0:
            raise B2SError(st, "b2s_ctx_create failed" + (" (no sm_90 GPU visible)" if st == 17 else ""))
        self.h = h
        self.curve = curve
        sz = (c_uint32 * 6)()
        self.lib.b2s_sizes(self.h, sz)
        self.fr_bytes, self.fq_bytes, self.g1_bytes, self.g2_bytes, self.g1x_bytes, self.g2x_bytes = list(sz)

    def close(self):
        if self.h:
            self.lib.b2s_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, st):
        if st != 0:
            raise B2SError(st, self.lib.b2s_last_error(self.h).decode())

    @property
    def launches(self):
        return int(self.lib.b2s_launch_count(self.h))

    @property
    def stream(self):
        return self.lib.b2s_stream(self.h)

    def sync(self):
        self._ck(self.lib.b2s_sync(self.h))

    # ---- kernels ------------------------------------------------------------------------------
    def ntt(self, data, log_n, inverse=False, coset=False):
        p, mem = _ptr(data)
        self._ck(self.lib.b2s_ntt(self.h, p, log_n, int(inverse), int(coset), mem))
        return data

    def _msm(self, fn, out_bytes, bases, scalars, n, mont):
        (pb, ps), mem = _ptrs(bases, scalars, same=n != 0)
        out = np.zeros(out_bytes // 4, dtype=np.uint32)
        self._ck(fn(self.h, pb, ps, n, int(mont), mem, out.ctypes.data))
        return out

    def msm_g1(self, bases, scalars, n, mont=True):
        return self._msm(self.lib.b2s_msm_g1, self.g1_bytes, bases, scalars, n, mont)

    def msm_g2(self, bases, scalars, n, mont=True):
        return self._msm(self.lib.b2s_msm_g2, self.g2_bytes, bases, scalars, n, mont)

    def msm_g1_partial(self, bases, scalars, n, mont=True):
        return self._msm(self.lib.b2s_msm_g1_partial, self.g1x_bytes, bases, scalars, n, mont)

    def msm_g2_partial(self, bases, scalars, n, mont=True):
        return self._msm(self.lib.b2s_msm_g2_partial, self.g2x_bytes, bases, scalars, n, mont)

    def g1_sum(self, xyzz, count):
        out = np.zeros(self.g1_bytes // 4, dtype=np.uint32)
        self._ck(self.lib.b2s_g1_sum(self.h, xyzz.ctypes.data, count, out.ctypes.data))
        return out

    def g2_sum(self, xyzz, count):
        out = np.zeros(self.g2_bytes // 4, dtype=np.uint32)
        self._ck(self.lib.b2s_g2_sum(self.h, xyzz.ctypes.data, count, out.ctypes.data))
        return out

    def fixed_base(self, group, scalars, n, mont=True, out=None):
        nbytes = (self.g1_bytes if group == 1 else self.g2_bytes) * n
        if out is None:
            assert _ptr(scalars)[1] == MEM_HOST
            out = np.zeros(nbytes // 4, dtype=np.uint32)
        (ps, po), mem = _ptrs(scalars, out)
        fn = self.lib.b2s_fixed_base_g1 if group == 1 else self.lib.b2s_fixed_base_g2
        self._ck(fn(self.h, ps, n, int(mont), mem, po))
        return out

    def field_op(self, field, op, a, b):
        out = np.zeros_like(a)
        limbs = (self.fq_bytes if field == 0 else self.fr_bytes) // 4
        self._ck(self.lib.b2s_field_op(self.h, field, op, a.ctypes.data, b.ctypes.data, out.ctypes.data, a.size // limbs))
        return out

    def group_op(self, group, op, a, b, k):
        out = np.zeros_like(a)
        limbs = (self.g1_bytes if group == 1 else self.g2_bytes) // 4
        self._ck(self.lib.b2s_group_op(self.h, group, op, a.ctypes.data, b.ctypes.data, k.ctypes.data, out.ctypes.data,
                                       a.size // limbs))
        return out

    # ---- R1CS ---------------------------------------------------------------------------------
    def r1cs_upload(self, n_rows, n_instance, n_witness, csr):
        """csr: three (row_ptr uint64[n_rows+1], col uint32[nnz], coeff uint32[nnz*8]) numpy triples."""
        rp = (c_void_p * 3)(*[m[0].ctypes.data for m in csr])
        col = (c_void_p * 3)(*[m[1].ctypes.data for m in csr])
        co = (c_void_p * 3)(*[m[2].ctypes.data for m in csr])
        h = c_void_p()
        self._ck(self.lib.b2s_r1cs_upload(self.h, n_rows, n_instance, n_witness, rp, col, co, ctypes.byref(h)))
        self._r1cs_vars[h.value] = n_instance + n_witness
        return h

    def r1cs_upload_lcmap(self, n_rows, n_instance, n_witness, args, lc_offsets, lc_vars, lc_coeffs, pool, outline=False):
        """The same handle, CSR built on the device from the constraint system's LcMap.  args: three uint64[n_rows] arrays
        of raw Variables; lc_offsets uint64[n_lcs+1]; lc_vars uint64[], lc_coeffs uint32[]; pool uint32[pool_len*8].
        outline=True: b2s_r1cs_upload_lcmap_outline, the instance variables outlined by outline_r1cs (n_instance more
        witnesses and rows; convert assignments with outline_assignment)."""
        a = (c_void_p * 3)(*[x.ctypes.data for x in args])
        h = c_void_p()
        common = (self.h, n_rows, n_instance, n_witness, a, len(lc_offsets) - 1, lc_offsets.ctypes.data, lc_vars.ctypes.data,
                  lc_coeffs.ctypes.data, pool.ctypes.data, len(pool) // 8)
        if outline:
            self._ck(self.lib.b2s_r1cs_upload_lcmap_outline(*common, ctypes.byref(Outline(OUTLINE_R1CS, 0)), ctypes.byref(h)))
            self._r1cs_vars[h.value] = 2 * n_instance + n_witness
            self._r1cs_src_vars[h.value] = n_instance + n_witness
        else:
            self._ck(self.lib.b2s_r1cs_upload_lcmap(*common, ctypes.byref(h)))
            self._r1cs_vars[h.value] = n_instance + n_witness
        return h

    def r1cs_free(self, m):
        self._r1cs_vars.pop(m.value if isinstance(m, c_void_p) else m, None)
        self._r1cs_src_vars.pop(m.value if isinstance(m, c_void_p) else m, None)
        self.lib.b2s_r1cs_free(self.h, m)

    def domain_size(self, m):
        return int(self.lib.b2s_r1cs_domain_size(m))

    def spmv(self, m, z, n_rows):
        pz, mem = _ptr(z)
        assert mem == MEM_HOST
        outs = [np.zeros(n_rows * 8, dtype=np.uint32) for _ in range(3)]
        self._ck(self.lib.b2s_spmv(self.h, m, pz, mem, *[o.ctypes.data for o in outs]))
        return outs

    def witness_map(self, m, z, qap=QAP_LIBSNARK):
        """h of the reduction `qap` (domain_size elements): libsnark coefficients, or circom odd-coset evaluations."""
        pz, mem = _ptr(z)
        assert mem == MEM_HOST
        h = np.zeros(self.domain_size(m) * 8, dtype=np.uint32)
        if qap == QAP_LIBSNARK:
            self._ck(self.lib.b2s_witness_map(self.h, m, pz, mem, h.ctypes.data))
        else:
            self._ck(self.lib.b2s_witness_map_qap(self.h, m, pz, mem, qap, h.ctypes.data))
        return h

    def witness_map_sim(self, m, z, log_ranks):
        """witness_map by the distributed schedule with 2^log_ranks virtual ranks on this GPU (test entry)."""
        pz, mem = _ptr(z)
        assert mem == MEM_HOST
        h = np.zeros(self.domain_size(m) * 8, dtype=np.uint32)
        self._ck(self.lib.b2s_witness_map_sim(self.h, m, pz, mem, log_ranks, h.ctypes.data))
        return h

    # ---- constraint satisfaction (ConstraintSystem::which_is_unsatisfied on the GPU) --------------------------------
    def gr1cs_upload(self, n_instance, n_witness, predicates):
        """predicates: {label: (arity, terms, matrices)}: terms [(coeff, [(argument, exponent), ...])] as
        ConstraintSystem.register_predicate takes them (constraint satisfied iff the polynomial is 0), matrices the predicate's
        `arity` matrices as to_matrices_all returns them (rows of (coeff, col)); Python ints.  Uploaded in sorted label order,
        the reference's BTreeMap order.  Returns a Gr1cs."""
        r = FR_MODULUS[self.curve]
        labels = sorted(predicates)
        descs = (PredicateDesc * max(len(labels), 1))()
        keep = []
        for d, label in zip(descs, labels):
            arity, terms, mats = predicates[label]
            d.arity, d.n_terms, d.n_rows = arity, len(terms), len(mats[0]) if mats else 0
            _set_poly(d, r, terms, keep)
            for j, m in enumerate(mats[:GR1CS_MAX_ARITY]):
                csr = _csr(r, m)
                keep += csr
                d.row_ptr[j], d.col[j], d.coeff[j] = (a.ctypes.data for a in csr)
        h = c_void_p()
        self._ck(self.lib.b2s_gr1cs_upload(self.h, n_instance, n_witness, len(labels), descs, ctypes.byref(h)))
        return Gr1cs(h, labels, n_instance + n_witness)

    def gr1cs_upload_lcmap(self, n_instance, n_witness, predicates, lcmap, outline=None):
        """The same Gr1cs, built on the device from the constraint system's LcMap.  predicates: {label: (arity, terms)} as for
        gr1cs_upload without the matrices; lcmap: the flat storage of every predicate -- offsets (n_lcs + 1), vars
        (raw Variables), coeffs (ids into pool), pool (Python ints, pool[0] = 1) and args {label: one sequence of raw Variables
        per argument, one Variable per constraint}; lists or numpy arrays.  Uploaded in sorted label order.
        outline=(strategy, label): b2s_gr1cs_upload_lcmap_outline, the instance variables outlined as finalize() does with an
        InstanceOutliner of that strategy (OUTLINE_R1CS / OUTLINE_SR1CS) whose tie rows go to predicate `label`; n_instance and
        n_witness are the counts before outlining.  Convert assignments with outline_assignment."""
        r = FR_MODULUS[self.curve]
        labels = sorted(predicates)
        descs = (PredicateLcmapDesc * max(len(labels), 1))()
        keep = []
        for d, label in zip(descs, labels):
            arity, terms = predicates[label]
            args = [np.ascontiguousarray(a, dtype=np.uint64) for a in lcmap["args"][label]]
            keep += args
            d.arity, d.n_terms, d.n_rows = arity, len(terms), len(args[0]) if args else 0
            _set_poly(d, r, terms, keep)
            for j, a in enumerate(args[:GR1CS_MAX_ARITY]):
                d.args[j] = a.ctypes.data
        off = np.ascontiguousarray(lcmap["offsets"], dtype=np.uint64)
        lc_vars = np.ascontiguousarray(lcmap["vars"], dtype=np.uint64)
        lc_coeffs = np.ascontiguousarray(lcmap["coeffs"], dtype=np.uint32)
        pool = _mont_limbs(r, lcmap["pool"])
        h = c_void_p()
        common = (self.h, n_instance, n_witness, len(labels), descs, len(off) - 1, off.ctypes.data, lc_vars.ctypes.data, lc_coeffs.ctypes.data,
                  pool.ctypes.data, len(lcmap["pool"]))
        if outline is None:
            self._ck(self.lib.b2s_gr1cs_upload_lcmap(*common, ctypes.byref(h)))
            return Gr1cs(h, labels, n_instance + n_witness)
        strategy, label = outline
        pred = labels.index(label) if label in labels else len(labels)
        self._ck(self.lib.b2s_gr1cs_upload_lcmap_outline(*common, ctypes.byref(Outline(strategy, pred)), ctypes.byref(h)))
        return Gr1cs(h, labels, 2 * n_instance + n_witness, n_instance + n_witness)

    def gr1cs_free(self, g):
        self.lib.b2s_gr1cs_free(self.h, g.h)

    def _check(self, fn, handle, n_pred, n_vars, z, counts):
        """z: (n_assign, n_vars * 8) 32-bit numpy array or CUDA torch tensor -> (first, count) uint64 numpy arrays of shape
        (n_assign, n_pred); count is None when counts=False (n_unsat = NULL).  The library reads n_assign * n_vars elements
        from z, so its shape is checked first."""
        width_ok = len(z.shape) == 2 and z.shape[1] == 8 * n_vars
        size_ok = (z.itemsize if isinstance(z, np.ndarray) else z.element_size()) == 4
        if not (width_ok and size_ok):
            raise ValueError(f"z must be (n_assign, {8 * n_vars}) 32-bit limbs for {n_vars} variables, got shape {tuple(z.shape)}")
        pz, mem = _ptr(z)
        n = z.shape[0]
        first, *count = _zeros([(n, n_pred)] * (2 if counts else 1), np.uint64, mem, z)
        count = count[0] if counts else None
        self._ck(fn(self.h, handle, n, pz, mem, _ptr(first)[0], _ptr(count)[0] if counts else None))
        if mem == MEM_DEVICE:
            first = first.cpu().numpy().view(np.uint64)
            count = count.cpu().numpy().view(np.uint64) if counts else None
        return first, count

    def gr1cs_check(self, g, z, counts=True):
        """b2s_gr1cs_check: first[i, p] = the first constraint of predicate g.labels[p] that assignment i does not satisfy
        (NOT_FOUND if none), count[i, p] how many it does not satisfy.  z: (n_assign, n_vars * 8) uint32 Montgomery limbs,
        HOST numpy or CUDA torch tensor."""
        return self._check(self.lib.b2s_gr1cs_check, g.h, len(g.labels), g.n_vars, z, counts)

    def r1cs_check(self, m, z, counts=True):
        """b2s_r1cs_check: the same for the R1CS predicate x0 * x1 - x2 of a Groth16 matrix handle (from r1cs_upload or
        r1cs_upload_lcmap of this Backend, which record its n_vars); arrays of shape (n_assign, 1)."""
        n_vars = self._r1cs_vars.get(m.value if isinstance(m, c_void_p) else m)
        if n_vars is None:
            raise ValueError("r1cs_check: not a live matrix handle of this Backend")
        return self._check(self.lib.b2s_r1cs_check, m, 1, n_vars, z, counts)

    def which_is_unsatisfied(self, g, z):
        """ConstraintSystem::which_is_unsatisfied for one assignment z (n_vars * 8 limbs): None, or (label, index) of the first
        unsatisfied constraint in label order."""
        first, _ = self.gr1cs_check(g, np.ascontiguousarray(z).reshape(1, -1), counts=False)
        for label, f in zip(g.labels, first[0]):
            if f != NOT_FOUND:
                return label, int(f)
        return None

    # ---- R1CS -> square R1CS (Sr1csAdapter) -----------------------------------------------------------------------------
    def r1cs_to_sr1cs(self, m):
        """b2s_r1cs_to_sr1cs: the square R1CS of a matrix handle of this Backend as a Gr1cs with the one predicate "SR1CS"
        (x0^2 - x1).  The source handle may be freed afterwards."""
        src_vars = self._r1cs_vars.get(m.value if isinstance(m, c_void_p) else m)
        if src_vars is None:
            raise ValueError("r1cs_to_sr1cs: not a live matrix handle of this Backend")
        h = c_void_p()
        self._ck(self.lib.b2s_r1cs_to_sr1cs(self.h, m, ctypes.byref(h)))
        info = self.gr1cs_info(Gr1cs(h, ["SR1CS"], 0))
        return Gr1cs(h, ["SR1CS"], info["n_instance"] + info["n_witness"], src_vars)

    def sr1cs_assignment(self, g, z, out=None):
        """b2s_sr1cs_assignment: z (n_assign, src_vars * 8) 32-bit limbs of the source's assignments, HOST numpy or CUDA
        torch tensor -> the converted assignments (n_assign, g.n_vars * 8) in the same memory (written into `out` if given)."""
        width = 8 * (g.src_vars or 0)
        if len(z.shape) != 2 or z.shape[1] != width:
            raise ValueError(f"z must be (n_assign, {width}) 32-bit limbs, got shape {tuple(z.shape)}")
        if out is None:
            if isinstance(z, np.ndarray):
                out = np.zeros((z.shape[0], 8 * g.n_vars), dtype=np.uint32)
            else:
                import torch

                out = torch.zeros((z.shape[0], 8 * g.n_vars), dtype=z.dtype, device=z.device)
                torch.cuda.current_stream(z.device).synchronize()
        (pz, po), mem = _ptrs(z, out)
        self._ck(self.lib.b2s_sr1cs_assignment(self.h, g.h, z.shape[0], pz, mem, po))
        return out

    def outline_assignment(self, h, z, out=None):
        """b2s_gr1cs_outline_assignment (h a Gr1cs) / b2s_r1cs_outline_assignment (h a matrix handle) of an outlined upload:
        z (n_assign, src_vars * 8) 32-bit limbs of assignments before outlining, HOST numpy or CUDA torch tensor -> the
        outlined assignments z || (ONE, z[1], ..., z[n_instance - 1]), (n_assign, n_vars * 8) in the same memory (written into
        `out` if given)."""
        if isinstance(h, Gr1cs):
            fn, handle, src, n_vars = self.lib.b2s_gr1cs_outline_assignment, h.h, h.src_vars or 0, h.n_vars
        else:
            key = h.value if isinstance(h, c_void_p) else h
            fn, handle, src, n_vars = self.lib.b2s_r1cs_outline_assignment, h, self._r1cs_src_vars.get(key, 0), self._r1cs_vars.get(key, 0)
        if len(z.shape) != 2 or z.shape[1] != 8 * src:
            raise ValueError(f"z must be (n_assign, {8 * src}) 32-bit limbs, got shape {tuple(z.shape)}")
        if out is None:
            if isinstance(z, np.ndarray):
                out = np.zeros((z.shape[0], 8 * n_vars), dtype=np.uint32)
            else:
                import torch

                out = torch.zeros((z.shape[0], 8 * n_vars), dtype=z.dtype, device=z.device)
                torch.cuda.current_stream(z.device).synchronize()
        (pz, po), mem = _ptrs(z, out)
        self._ck(fn(self.h, handle, z.shape[0], pz, mem, po))
        return out

    def gr1cs_info(self, g):
        """b2s_gr1cs_info: {"n_instance", "n_witness", "predicates": [(arity, n_rows, [nnz per argument])]} of any Gr1cs."""
        n_vars = (c_uint64 * 2)()
        n_pred = c_uint32()
        self._ck(self.lib.b2s_gr1cs_info(self.h, g.h, n_vars, ctypes.byref(n_pred), None, 0))
        preds = (Gr1csPredInfo * max(n_pred.value, 1))()
        self._ck(self.lib.b2s_gr1cs_info(self.h, g.h, n_vars, ctypes.byref(n_pred), preds, n_pred.value))
        return {"n_instance": int(n_vars[0]), "n_witness": int(n_vars[1]),
                "predicates": [(p.arity, int(p.n_rows), [int(x) for x in p.nnz[:p.arity]]) for p in preds[:n_pred.value]]}

    def gr1cs_export(self, g, pred, arg, info=None):
        """b2s_gr1cs_export: argument `arg` of predicate `pred` -> (row_ptr uint64[n_rows + 1], col uint32[nnz], coeff
        uint32[nnz * 8] Montgomery limbs)."""
        info = info or self.gr1cs_info(g)
        n_rows, nnz = 0, 0
        if pred < len(info["predicates"]):
            _, n_rows, nnzs = info["predicates"][pred]
            nnz = nnzs[arg] if arg < len(nnzs) else 0
        row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
        col = np.zeros(max(nnz, 1), dtype=np.uint32)
        coeff = np.zeros(max(nnz, 1) * 8, dtype=np.uint32)
        self._ck(self.lib.b2s_gr1cs_export(self.h, g.h, pred, arg, row_ptr.ctypes.data, row_ptr.nbytes, col.ctypes.data, 4 * nnz,
                                           coeff.ctypes.data, 32 * nnz))
        return row_ptr, col[:nnz], coeff[:8 * nnz]

    # ---- Groth16 ------------------------------------------------------------------------------
    def pk_upload(self, desc: PkDesc, mem=MEM_HOST, qap=QAP_LIBSNARK):
        h = c_void_p()
        if qap == QAP_LIBSNARK:
            self._ck(self.lib.b2s_pk_upload(self.h, ctypes.byref(desc), mem, ctypes.byref(h)))
        else:
            self._ck(self.lib.b2s_pk_upload_qap(self.h, ctypes.byref(desc), mem, qap, ctypes.byref(h)))
        return h

    def groth16_setup(self, m, trapdoor, n_instance, qap=QAP_LIBSNARK):
        """trapdoor: uint32[5*8] Montgomery (tau, alpha, beta, gamma, delta) -> (pk handle, vk dict of numpy arrays).
        qap: the key's reduction (QAP_CIRCOM: the N-point circom h query)."""
        h = c_void_p()
        vk = self._vk_bufs(n_instance)
        outs = [v.ctypes.data for v in vk.values()]
        if qap == QAP_LIBSNARK:
            self._ck(self.lib.b2s_groth16_setup(self.h, m, trapdoor.ctypes.data, ctypes.byref(h), *outs))
        else:
            self._ck(self.lib.b2s_groth16_setup_qap(self.h, m, trapdoor.ctypes.data, qap, ctypes.byref(h), *outs))
        return h, vk

    def _vk_bufs(self, n_abc):
        """A zeroed verifying key: the dict of HOST arrays groth16_setup returns, with room for max(n_abc, 1) gamma_abc_g1
        points; the values are in the order of the C ABI's vk arguments."""
        g1, g2 = (np.zeros(n // 4, dtype=np.uint32) for n in (self.g1_bytes, self.g2_bytes))
        return {"alpha_g1": g1, "beta_g2": g2, "gamma_g2": g2.copy(), "delta_g2": g2.copy(),
                "gamma_abc_g1": np.zeros(max(n_abc, 1) * self.g1_bytes // 4, dtype=np.uint32)}

    def pk_query(self, pk, which, count):
        per = self.g2_bytes if which in (2, 6) else self.g1_bytes
        out = np.zeros(count * per // 4, dtype=np.uint32)
        self._ck(self.lib.b2s_pk_query(self.h, pk, which, out.ctypes.data, out.nbytes))
        return out

    def serialize_points(self, group, affine, count, compressed=True):
        per = (self.fq_bytes if group == 1 else 2 * self.fq_bytes) * (1 if compressed else 2)
        out = np.zeros(count * per, dtype=np.uint8)
        name = f"b2s_serialize_g{group}_{'compressed' if compressed else 'uncompressed'}"
        self._ck(getattr(self.lib, name)(self.h, affine.ctypes.data, count, out.ctypes.data, out.nbytes))
        return out.tobytes()

    def proof_bytes(self, a, b, c, compressed=True):
        out = np.zeros(4 * self.fq_bytes * (1 if compressed else 2), dtype=np.uint8)
        fn = self.lib.b2s_proof_serialize_compressed if compressed else self.lib.b2s_proof_serialize_uncompressed
        self._ck(fn(self.h, a.ctypes.data, b.ctypes.data, c.ctypes.data, out.ctypes.data, out.nbytes))
        return out.tobytes()

    def vk_bytes(self, alpha_g1, beta_g2, gamma_g2, delta_g2, gamma_abc_g1, n_gamma_abc, compressed=True):
        """ark-groth16 VerifyingKey bytes from the HOST affine points b2s_groth16_setup returned."""
        out = np.zeros(int(self.lib.b2s_vk_serialized_size(self.h, n_gamma_abc, int(compressed))), dtype=np.uint8)
        self._ck(self.lib.b2s_vk_serialize(self.h, alpha_g1.ctypes.data, beta_g2.ctypes.data, gamma_g2.ctypes.data, delta_g2.ctypes.data,
                                           gamma_abc_g1.ctypes.data, n_gamma_abc, int(compressed), out.ctypes.data, out.nbytes))
        return out.tobytes()

    def pk_bytes(self, pk, vk_bytes, compressed=True):
        """ark-groth16 ProvingKey bytes of a device-resident full key (vk_bytes from vk_bytes())."""
        vk = np.frombuffer(vk_bytes, dtype=np.uint8)
        out = np.zeros(int(self.lib.b2s_pk_serialized_size(self.h, pk, len(vk), int(compressed))), dtype=np.uint8)
        self._ck(self.lib.b2s_pk_serialize(self.h, pk, vk.ctypes.data, len(vk), int(compressed), out.ctypes.data, out.nbytes))
        return out.tobytes()

    # ---- CanonicalDeserialize (decoding and validation on the GPU) ------------------------------------------------
    def deserialize_points(self, group, data, count=None, compressed=True, validate=True):
        """`count` encoded points (default: as many as `data` holds) -> HOST affine Montgomery limbs (uint32)."""
        per = (self.fq_bytes if group == 1 else 2 * self.fq_bytes) * (1 if compressed else 2)
        buf = np.frombuffer(bytes(data), dtype=np.uint8)
        count = len(buf) // per if count is None else count
        out = np.zeros(max(count, 1) * (self.g1_bytes if group == 1 else self.g2_bytes) // 4, dtype=np.uint32)
        fn = self.lib.b2s_deserialize_g1 if group == 1 else self.lib.b2s_deserialize_g2
        self._ck(fn(self.h, buf.ctypes.data, len(buf), count, int(compressed), int(validate), out.ctypes.data))
        return out[: count * (self.g1_bytes if group == 1 else self.g2_bytes) // 4]

    def proof_from_bytes(self, data, compressed=True, validate=True):
        """Proof bytes -> (a, b, c) HOST affine arrays, the layout groth16_prove returns."""
        buf = np.frombuffer(bytes(data), dtype=np.uint8)
        a, b, c = self._proof_bufs()
        self._ck(self.lib.b2s_proof_deserialize(self.h, buf.ctypes.data, len(buf), int(compressed), int(validate), a.ctypes.data,
                                                b.ctypes.data, c.ctypes.data))
        return a, b, c

    def vk_from_bytes(self, data, compressed=True, validate=True):
        """VerifyingKey from the start of `data` -> (vk dict in the layout groth16_setup returns, bytes consumed)."""
        buf = np.frombuffer(bytes(data), dtype=np.uint8)
        n, used = c_uint64(), c_uint64()
        self._ck(self.lib.b2s_vk_deserialize(self.h, buf.ctypes.data, len(buf), int(compressed), int(validate), None, None, None, None,
                                             None, 0, ctypes.byref(n), ctypes.byref(used)))
        vk = self._vk_bufs(n.value)
        self._ck(self.lib.b2s_vk_deserialize(self.h, buf.ctypes.data, len(buf), int(compressed), int(validate),
                                             *(v.ctypes.data for v in vk.values()), n.value, ctypes.byref(n), ctypes.byref(used)))
        vk["gamma_abc_g1"] = vk["gamma_abc_g1"][: n.value * self.g1_bytes // 4]
        return vk, used.value

    def pk_from_bytes(self, data, compressed=True, validate=True, qap=QAP_LIBSNARK):
        """ark-groth16 ProvingKey bytes -> device-resident full key handle (as pk_upload returns).  qap=QAP_CIRCOM reads the
        bytes of a Groth16<E, CircomReduction> key (|h_query| = domain size)."""
        buf = np.frombuffer(bytes(data), dtype=np.uint8)
        h = c_void_p()
        if qap == QAP_LIBSNARK:
            self._ck(self.lib.b2s_pk_deserialize(self.h, buf.ctypes.data, len(buf), int(compressed), int(validate), ctypes.byref(h)))
        else:
            self._ck(self.lib.b2s_pk_deserialize_qap(self.h, buf.ctypes.data, len(buf), int(compressed), int(validate), qap,
                                                     ctypes.byref(h)))
        return h

    def pk_free(self, pk):
        self.lib.b2s_pk_free(self.h, pk)

    # ---- snarkjs and circom files (.zkey / .wtns / .r1cs) ------------------------------------------------------------
    @staticmethod
    def _file_bytes(data):
        """bytes-like or numpy array (an np.memmap of the file included) -> a uint8 view of the same memory, not a copy"""
        if isinstance(data, np.ndarray):
            assert data.flags["C_CONTIGUOUS"]
            return data.reshape(-1).view(np.uint8)
        return np.frombuffer(data, dtype=np.uint8)

    def zkey_info(self, data):
        """Header of a snarkjs Groth16 .zkey: {n_vars, n_public, domain_size, n_coeffs}."""
        buf = self._file_bytes(data)
        info = ZkeyInfo()
        self._ck(self.lib.b2s_zkey_read_info(self.h, buf.ctypes.data, buf.nbytes, ctypes.byref(info)))
        return {name: int(getattr(info, name)) for name, _ in ZkeyInfo._fields_}

    def zkey_load(self, data, validate=True):
        """A snarkjs Groth16 .zkey (bytes, or a numpy array / np.memmap of the file) -> (pk, m, vk): the device-resident
        circom key, the matrix handle (A and B, C empty) and the verifying key in the layout vk_from_bytes returns."""
        buf = self._file_bytes(data)
        info = self.zkey_info(buf)
        n_abc = info["n_public"] + 1
        vk = self._vk_bufs(n_abc)
        pk, m = c_void_p(), c_void_p()
        self._ck(self.lib.b2s_zkey_load(self.h, buf.ctypes.data, buf.nbytes, int(validate), ctypes.byref(pk), ctypes.byref(m),
                                        *(v.ctypes.data for v in vk.values()), n_abc))
        self._r1cs_vars[m.value] = info["n_vars"]
        return pk, m, vk

    def wtns_read(self, data, n_vars, out=None):
        """A circom .wtns -> z = instance || witness, n_vars Montgomery Fr: a new uint32 numpy array, or written into `out`
        (a host numpy array, or a CUDA torch tensor / device address, e.g. one row of a prove_batch z) and returned."""
        buf = self._file_bytes(data)
        if out is None:
            out = np.zeros(n_vars * self.fr_bytes // 4, dtype=np.uint32)
        po, mem = _ptr(out)
        self._ck(self.lib.b2s_wtns_read(self.h, buf.ctypes.data, buf.nbytes, n_vars, mem, po))
        return out

    def r1cs_file_info(self, data):
        """Header of a circom .r1cs (bytes, or a numpy array / np.memmap of the file): {n_wires, n_pub_out, n_pub_in, n_prv_in,
        n_labels, n_constraints, domain_size}."""
        buf = self._file_bytes(data)
        info = R1csFileInfo()
        self._ck(self.lib.b2s_r1cs_file_read_info(self.h, buf.ctypes.data, buf.nbytes, ctypes.byref(info)))
        return {name: int(getattr(info, name)) for name, _ in R1csFileInfo._fields_}

    def r1cs_file_load(self, data):
        """A circom .r1cs (bytes, or a numpy array / np.memmap of the file) -> the matrix handle r1cs_upload builds from the
        same A, B, C (n_instance = 1 + n_pub_out + n_pub_in), checked and decoded on the GPU."""
        buf = self._file_bytes(data)
        info = self.r1cs_file_info(buf)
        m = c_void_p()
        self._ck(self.lib.b2s_r1cs_file_load(self.h, buf.ctypes.data, buf.nbytes, ctypes.byref(m)))
        self._r1cs_vars[m.value] = info["n_wires"]
        return m

    # ---- verification (pairings in CUDA) ----------------------------------------------------------------------------
    def vk_prepare(self, vk):
        """vk dict in the layout groth16_setup / vk_from_bytes return (HOST arrays) -> device-resident prepared key handle."""
        n_abc = len(vk["gamma_abc_g1"]) * 4 // self.g1_bytes
        h = c_void_p()
        self._ck(self.lib.b2s_vk_prepare(self.h, vk["alpha_g1"].ctypes.data, vk["beta_g2"].ctypes.data, vk["gamma_g2"].ctypes.data,
                                         vk["delta_g2"].ctypes.data, vk["gamma_abc_g1"].ctypes.data if n_abc else None, n_abc,
                                         ctypes.byref(h)))
        return h

    def pvk_free(self, pvk):
        self.lib.b2s_pvk_free(self.h, pvk)

    def groth16_verify_batch(self, pvk, inputs, n_inputs, a, b, c, n_proofs=None, ok=None):
        """One verdict per proof.  inputs: n_proofs x n_inputs Montgomery Fr (None when n_inputs == 0); a, b, c: affine
        arrays; all HOST numpy or all CUDA torch tensors.  Returns a bool numpy array (host), or fills the uint8 tensor
        `ok` (device) and returns it."""
        (pa, pb, pc, px), mem = _ptrs(a, b, c, inputs)
        if n_proofs is None:
            n_proofs = _nbytes(a) // self.g1_bytes
        if mem == MEM_HOST:
            out = np.zeros(max(n_proofs, 1), dtype=np.uint8)
            self._ck(self.lib.b2s_groth16_verify_batch(self.h, pvk, n_proofs, px, n_inputs, pa, pb, pc, mem, out.ctypes.data))
            return out[:n_proofs].astype(bool)
        po, _ = _ptr(ok)
        self._ck(self.lib.b2s_groth16_verify_batch(self.h, pvk, n_proofs, px, n_inputs, pa, pb, pc, mem, po))
        return ok

    def groth16_verify_all(self, pvk, inputs, n_inputs, a, b, c, rho=None, n_proofs=None):
        """True when every proof is accepted, by one random linear combination of the batch (b2s_groth16_verify_batch_rlc).
        Buffers as for groth16_verify_batch.  rho: n_proofs x 4 uint32 words (little-endian 128-bit, nonzero) in the same
        memory as the proofs; None draws them with `secrets`.  On False, groth16_verify_batch tells which proofs failed."""
        (pa, pb, pc, px), mem = _ptrs(a, b, c, inputs)
        if n_proofs is None:
            n_proofs = _nbytes(a) // self.g1_bytes
        if rho is None:
            rho = _draw_rho(n_proofs, mem, a)
        pr, mem_r = _ptr(rho)
        assert n_proofs == 0 or mem_r == mem
        ok = ctypes.c_uint8(0)
        self._ck(self.lib.b2s_groth16_verify_batch_rlc(self.h, pvk, n_proofs, px, n_inputs, pa, pb, pc, pr, mem, ctypes.byref(ok)))
        return bool(ok.value)

    def _proof_buf(self, proofs, compressed, n_proofs):
        """serialized proofs (bytes / numpy uint8 on the HOST, or a CUDA torch uint8 tensor) -> (address, mem, len, n_proofs)"""
        if isinstance(proofs, (bytes, bytearray, memoryview)):
            proofs = np.frombuffer(bytes(proofs), dtype=np.uint8)
        ln = _nbytes(proofs)
        pp, mem = _ptr(proofs)
        if n_proofs is None:
            n_proofs = ln // (4 * self.fq_bytes * (1 if compressed else 2))
        return proofs, pp, mem, ln, n_proofs

    def groth16_verify_batch_bytes(self, pvk, inputs, n_inputs, proofs, compressed=True, n_proofs=None, ok=None, reason=None):
        """One verdict per ark-serialized proof (b2s_groth16_verify_batch_bytes): `proofs` is a || b || c per proof, back to
        back, decoded and validated on the GPU.  inputs as for groth16_verify_batch, in the same memory as `proofs`.  Returns
        (ok, reason): a bool and a uint8 numpy array for HOST buffers (reason[i] = 0 when proof i decoded, else
        16 (1 + element) + decode reason); for device buffers fills the uint8 tensors `ok` and `reason` (may be None)."""
        proofs, pp, mem, ln, n_proofs = self._proof_buf(proofs, compressed, n_proofs)
        px, mem_x = _ptr(inputs)
        assert inputs is None or mem_x == mem
        if mem == MEM_HOST:
            out, rs = np.zeros(max(n_proofs, 1), dtype=np.uint8), np.zeros(max(n_proofs, 1), dtype=np.uint8)
            self._ck(self.lib.b2s_groth16_verify_batch_bytes(self.h, pvk, n_proofs, px, n_inputs, pp, ln, int(compressed), mem,
                                                             out.ctypes.data, rs.ctypes.data))
            return out[:n_proofs].astype(bool), rs[:n_proofs]
        po, _ = _ptr(ok)
        pr, _ = _ptr(reason)
        self._ck(self.lib.b2s_groth16_verify_batch_bytes(self.h, pvk, n_proofs, px, n_inputs, pp, ln, int(compressed), mem, po, pr))
        return ok, reason

    def groth16_verify_all_bytes(self, pvk, inputs, n_inputs, proofs, compressed=True, rho=None, n_proofs=None, reason=None):
        """True when every ark-serialized proof decodes and the batch passes the random linear combination
        (b2s_groth16_verify_batch_rlc_bytes).  Buffers as for groth16_verify_batch_bytes; rho as for groth16_verify_all (None
        draws it with `secrets`).  Returns (verdict, reason): reason is a uint8 numpy array for HOST buffers, else the
        device tensor `reason` passed in (may be None)."""
        proofs, pp, mem, ln, n_proofs = self._proof_buf(proofs, compressed, n_proofs)
        px, mem_x = _ptr(inputs)
        assert inputs is None or mem_x == mem
        if rho is None:
            rho = _draw_rho(n_proofs, mem, proofs)
        pr, mem_r = _ptr(rho)
        assert n_proofs == 0 or mem_r == mem
        if mem == MEM_HOST:
            reason = np.zeros(max(n_proofs, 1), dtype=np.uint8)
        prs, _ = _ptr(reason)
        ok = ctypes.c_uint8(0)
        self._ck(self.lib.b2s_groth16_verify_batch_rlc_bytes(self.h, pvk, n_proofs, px, n_inputs, pp, ln, int(compressed), pr, mem,
                                                             ctypes.byref(ok), prs))
        return bool(ok.value), (reason[:n_proofs] if mem == MEM_HOST else reason)

    def pairing(self, p, q, n=None, out=None):
        """e(P_i, Q_i) element-wise.  p, q: affine G1 / G2 arrays (HOST numpy, or CUDA torch tensors with `out` a device
        tensor of n * 12 Fq).  Returns GT elements as uint32 limbs (ark's Fp12 layout, Montgomery)."""
        if n is None:
            n = _nbytes(p) // self.g1_bytes
        if out is None:
            assert _ptr(p)[1] == MEM_HOST
            out = np.zeros(n * 12 * self.fq_bytes // 4, dtype=np.uint32)
        (pp, pq, po), mem = _ptrs(p, q, out)
        self._ck(self.lib.b2s_pairing(self.h, pp, pq, n, mem, po))
        return out

    def _proof_bufs(self):
        return (np.zeros(self.g1_bytes // 4, dtype=np.uint32), np.zeros(self.g2_bytes // 4, dtype=np.uint32),
                np.zeros(self.g1_bytes // 4, dtype=np.uint32))

    def groth16_prove(self, pk, m, z_inst, z_wit, r, s):
        a, b, c = self._proof_bufs()
        self._ck(self.lib.b2s_groth16_prove(self.h, pk, m, _ptr(z_inst)[0], _ptr(z_wit)[0], r.ctypes.data, s.ctypes.data,
                                            a.ctypes.data, b.ctypes.data, c.ctypes.data))
        return a, b, c

    def groth16_prove_resident(self, pk, m, z_dev, r, s):
        a, b, c = self._proof_bufs()
        self._ck(self.lib.b2s_groth16_prove_resident(self.h, pk, m, _ptr(z_dev)[0], r.ctypes.data, s.ctypes.data,
                                                     a.ctypes.data, b.ctypes.data, c.ctypes.data))
        return a, b, c

    def groth16_prove_batch(self, pk, m, z, r, s):
        """n_proofs proofs under one key in one call (b2s_groth16_prove_batch).  z: n_proofs rows of n_instance + n_witness
        Montgomery Fr (row i = proof i's instance || witness); r, s: n_proofs Montgomery Fr each; all HOST numpy arrays or all
        CUDA torch tensors.  Returns (a, b, c): n_proofs x (G1 / G2 / G1 affine) uint32 numpy arrays, or int32 tensors on the
        device of the inputs (the library's stream is synchronised before return)."""
        (pz, pr, ps), mem = _ptrs(z, r, s)
        n = _nbytes(r) // self.fr_bytes
        w1, w2 = self.g1_bytes // 4, self.g2_bytes // 4
        a, b, c = _zeros([(n, w1), (n, w2), (n, w1)], np.uint32, mem, r)
        self._ck(self.lib.b2s_groth16_prove_batch(self.h, pk, m, n, pz, pr, ps, mem, _ptr(a)[0], _ptr(b)[0], _ptr(c)[0]))
        return a, b, c

    def groth16_prove_shard_resident(self, pk, m, z_dev, r, s):
        g1 = np.zeros(4 * self.g1x_bytes // 4, dtype=np.uint32)
        g2 = np.zeros(self.g2x_bytes // 4, dtype=np.uint32)
        self._ck(self.lib.b2s_groth16_prove_shard_resident(self.h, pk, m, _ptr(z_dev)[0], r.ctypes.data, s.ctypes.data,
                                                           g1.ctypes.data, g2.ctypes.data))
        return g1, g2

    def profile(self, on=True):
        self._ck(self.lib.b2s_profile_enable(self.h, int(on)))

    def profile_report(self):
        """{kernel name: (launches, total_ms)} since the last report."""
        buf = ctypes.create_string_buffer(1 << 16)
        self._ck(self.lib.b2s_profile_report(self.h, buf, len(buf)))
        out = {}
        for line in buf.value.decode().splitlines():
            name, cnt, ms = line.split("\t")
            out[name] = (int(cnt), float(ms))
        return out

    def groth16_prove_shard(self, pk, m, z_inst, z_wit, r, s):
        g1 = np.zeros(4 * self.g1x_bytes // 4, dtype=np.uint32)
        g2 = np.zeros(self.g2x_bytes // 4, dtype=np.uint32)
        self._ck(self.lib.b2s_groth16_prove_shard(self.h, pk, m, _ptr(z_inst)[0], _ptr(z_wit)[0], r.ctypes.data, s.ctypes.data,
                                                  g1.ctypes.data, g2.ctypes.data))
        return g1, g2

    # ---- multi-GPU group (NCCL inside the library) ----------------------------------------------
    @staticmethod
    def group_unique_id():
        """128-byte NCCL id (rank 0 draws it; the host program distributes it)."""
        buf = np.zeros(128, dtype=np.uint8)
        st = load_library().b2s_group_unique_id(buf.ctypes.data)
        if st != 0:
            raise B2SError(st, "b2s_group_unique_id failed (NCCL not loadable?)")
        return buf

    def group_create(self, uid, rank, world):
        g = c_void_p()
        uid = np.ascontiguousarray(uid, dtype=np.uint8) if uid is not None else None
        self._ck(self.lib.b2s_group_create(self.h, uid.ctypes.data if uid is not None else None, rank, world, ctypes.byref(g)))
        return g

    def group_destroy(self, g):
        self.lib.b2s_group_destroy(g)

    def groth16_prove_group(self, g, pk, m, z_inst, z_wit, r, s):
        """Collective over the group; the proof (a, b, c) is meaningful on rank 0."""
        a, b, c = self._proof_bufs()
        st = self.lib.b2s_groth16_prove_group(g, pk, m, _ptr(z_inst)[0], _ptr(z_wit)[0], r.ctypes.data, s.ctypes.data, a.ctypes.data,
                                              b.ctypes.data, c.ctypes.data)
        self._ck(st)
        return a, b, c

    def groth16_prove_group_resident(self, g, pk, m, z_dev, r, s):
        a, b, c = self._proof_bufs()
        st = self.lib.b2s_groth16_prove_group_resident(g, pk, m, _ptr(z_dev)[0], r.ctypes.data, s.ctypes.data, a.ctypes.data,
                                                       b.ctypes.data, c.ctypes.data)
        self._ck(st)
        return a, b, c

    def groth16_finish(self, pk, g1_partials, g2_partials, n_shards, r, s):
        a, b, c = self._proof_bufs()
        self._ck(self.lib.b2s_groth16_finish(self.h, pk, g1_partials.ctypes.data, g2_partials.ctypes.data, n_shards,
                                             r.ctypes.data, s.ctypes.data, a.ctypes.data, b.ctypes.data, c.ctypes.data))
        return a, b, c
