"""Writers of snarkjs's Groth16 .zkey and circom's .wtns files.  TEST INFRASTRUCTURE ONLY.

Restated from snarkjs's zkey / wtns writers (binfile framing, toRprLEM points, coefficients stored as c R^2 mod r, the
nPublic + 1 input rows appended to A) -- see snark_b200/csrc/zkey.cu for the layout.  Neither snarkjs nor ark-circom is in
the reference tree and no file written by snarkjs exists here, so these writers and the library's readers are checked for
consistency with each other only: byte parity with snarkjs is NOT pinned.

Points and coefficients are taken as C-ABI numpy arrays (Montgomery limbs, tests/util.py), so keys downloaded from the GPU
at 2^24 are written without Python-int loops: field values are converted once per distinct value.
"""
import struct

import numpy as np

ZKEY_SECTIONS = {"protocol": 1, "header": 2, "ic": 3, "coeffs": 4, "a": 5, "b1": 6, "b2": 7, "c": 8, "h": 9, "contributions": 10}


def _int_bytes(x, n):
    return int(x).to_bytes(n, "little")


def _limbs_to_int(row):
    return sum(int(w) << (32 * j) for j, w in enumerate(row))


def fr_rescale(curve, limbs, factor):
    """uint32[n * 8] field elements -> the same layout with every value v replaced by v * factor mod r (once per distinct v)"""
    rows = np.ascontiguousarray(limbs, dtype=np.uint32).reshape(-1, 8)
    if len(rows) == 0:
        return rows.reshape(-1)
    uniq, inv = np.unique(rows, axis=0, return_inverse=True)
    out = np.zeros_like(uniq)
    for i, row in enumerate(uniq):
        v = _limbs_to_int(row) * factor % curve.r
        out[i] = [(v >> (32 * j)) & 0xFFFFFFFF for j in range(8)]
    return out[np.asarray(inv).reshape(-1)].reshape(-1)


def key_arrays(curve, pk):
    """oracle ProvingKey (oracle/groth16.py, circom h query) -> the dict of packed arrays write_zkey takes"""
    from tests.util import pack_points

    g1 = lambda pts: pack_points(curve, 1, pts)
    g2 = lambda pts: pack_points(curve, 2, pts)
    return {"alpha_g1": g1([pk.alpha_g1]), "beta_g1": g1([pk.beta_g1]), "delta_g1": g1([pk.delta_g1]), "beta_g2": g2([pk.beta_g2]),
            "gamma_g2": g2([pk.gamma_g2]), "delta_g2": g2([pk.delta_g2]), "gamma_abc_g1": g1(pk.gamma_abc_g1), "a": g1(pk.a_query),
            "b_g1": g1(pk.b_g1_query), "b_g2": g2(pk.b_g2_query), "h": g1(pk.h_query), "l": g1(pk.l_query)}


def key_arrays_device(be, pkh, vk, n_instance, n_witness, domain):
    """the same dict from a device-resident circom key (Backend.groth16_setup(.., qap=QAP_CIRCOM)) and its vk"""
    n_vars = n_instance + n_witness
    c1, c2 = be.pk_query(pkh, 5, 3).reshape(3, -1), be.pk_query(pkh, 6, 2).reshape(2, -1)
    return {"alpha_g1": c1[0], "beta_g1": c1[1], "delta_g1": c1[2], "beta_g2": c2[0], "gamma_g2": vk["gamma_g2"], "delta_g2": c2[1],
            "gamma_abc_g1": vk["gamma_abc_g1"][: n_instance * be.g1_bytes // 4], "a": be.pk_query(pkh, 0, n_vars),
            "b_g1": be.pk_query(pkh, 1, n_vars), "b_g2": be.pk_query(pkh, 2, n_vars), "h": be.pk_query(pkh, 3, domain),
            "l": be.pk_query(pkh, 4, n_witness)}


def coeff_records(curve, csr_a, csr_b, n_public):
    """snarkjs's coefficient records, in its order (per constraint: A's entries, then B's; then the input rows
    A[n + s] = 1 * z[s]) as an (n_entries, 11) uint32 array: matrix, constraint, signal, value (c R^2 mod r, 8 limbs).
    csr_*: (row_ptr, col, Montgomery coefficient limbs) as tests/util.csr_from_rows returns them."""
    R = 1 << 256
    n = len(csr_a[0]) - 1
    parts = []
    for mat, (row_ptr, col, coeff) in enumerate((csr_a, csr_b)):
        rows = np.repeat(np.arange(n, dtype=np.uint32), np.diff(row_ptr.astype(np.int64)))
        rec = np.zeros((len(col), 11), dtype=np.uint32)
        rec[:, 0], rec[:, 1], rec[:, 2] = mat, rows, col
        rec[:, 3:] = fr_rescale(curve, coeff, R).reshape(-1, 8)   # c R -> c R^2
        parts.append(rec)
    rec = np.concatenate(parts)
    rec = rec[np.lexsort((rec[:, 0], rec[:, 1]))]   # by constraint, A before B, stable within a row
    inp = np.zeros((n_public + 1, 11), dtype=np.uint32)
    one = R * R % curve.r
    inp[:, 1] = n + np.arange(n_public + 1)
    inp[:, 2] = np.arange(n_public + 1)
    inp[:, 3:] = [(one >> (32 * j)) & 0xFFFFFFFF for j in range(8)]
    return np.concatenate([rec, inp])


def binfile(magic, version, sections):
    """magic, u32 version, u32 section count, then (u32 type, u64 size, bytes) per section, in the order given"""
    out = [magic, struct.pack("<II", version, len(sections))]
    for t, body in sections:
        out += [struct.pack("<IQ", t, len(body)), body]
    return b"".join(out)


def zkey_sections(curve, key, records, n_public, domain, protocol=1):
    """[(type, bytes)] of a Groth16 zkey in snarkjs's order (1..9); `key` as key_arrays returns it"""
    n8q, n8r = 8 * curve.fq_limbs64, 32
    n_vars = len(key["a"]) * 4 // (2 * n8q)
    b = lambda a: np.ascontiguousarray(a, dtype=np.uint32).tobytes()
    header = (struct.pack("<I", n8q) + _int_bytes(curve.p, n8q) + struct.pack("<I", n8r) + _int_bytes(curve.r, n8r)
              + struct.pack("<III", n_vars, n_public, domain)
              + b"".join(b(key[k]) for k in ("alpha_g1", "beta_g1", "beta_g2", "gamma_g2", "delta_g1", "delta_g2")))
    coeffs = struct.pack("<I", len(records)) + np.ascontiguousarray(records, dtype=np.uint32).tobytes()
    return [(1, struct.pack("<I", protocol)), (2, header), (3, b(key["gamma_abc_g1"])), (4, coeffs), (5, b(key["a"])), (6, b(key["b_g1"])),
            (7, b(key["b_g2"])), (8, b(key["l"])), (9, b(key["h"]))]


def write_zkey(curve, key, csr_a, csr_b, n_public, domain, order="snarkjs", seed=0, protocol=1):
    """A Groth16 .zkey of the circom key `key` (key_arrays / key_arrays_device) and the matrices A, B (CSR, Montgomery).
    order="snarkjs": sections 1..9 and records as snarkjs writes them; "shuffled": records and sections permuted, with a
    contributions section (10) and an unknown section added."""
    rec = coeff_records(curve, csr_a, csr_b, n_public)
    secs = None
    if order == "shuffled":
        rng = np.random.default_rng(seed)
        rec = rec[rng.permutation(len(rec))]
        secs = zkey_sections(curve, key, rec, n_public, domain, protocol)
        secs += [(10, b"\x07" * 40), (77, b"unknown section")]
        secs = [secs[i] for i in rng.permutation(len(secs))]
    else:
        assert order == "snarkjs", order
        secs = zkey_sections(curve, key, rec, n_public, domain, protocol)
    return binfile(b"zkey", 1, secs)


def write_wtns(curve, z, mont=True):
    """A .wtns of z = instance || witness: z as C-ABI limbs (Montgomery when mont, else canonical) or a list of ints"""
    if isinstance(z, np.ndarray):
        vals = fr_rescale(curve, z, pow(1 << 256, -1, curve.r)) if mont else np.ascontiguousarray(z, dtype=np.uint32).reshape(-1)
        data = vals.tobytes()
        n = len(vals) // 8
    else:
        data = b"".join(_int_bytes(v % curve.r, 32) for v in z)
        n = len(z)
    return binfile(b"wtns", 2, [(1, struct.pack("<I", 32) + _int_bytes(curve.r, 32) + struct.pack("<I", n)), (2, data)])
