"""Shared helpers for the tests: limb packing between Python ints and the C-ABI layout."""
import ctypes

import numpy as np


def pack_u32(xs, n):
    """ints -> contiguous uint32 array of len(xs)*n little-endian limbs."""
    arr = np.zeros(len(xs) * n, dtype=np.uint32)
    for i, x in enumerate(xs):
        for j in range(n):
            arr[i * n + j] = (x >> (32 * j)) & 0xFFFFFFFF
    return arr


def unpack_u32(arr, n):
    arr = np.asarray(arr, dtype=np.uint32).reshape(-1, n)
    return [sum(int(row[j]) << (32 * j) for j in range(n)) for row in arr]


def ptr(a, ty=ctypes.c_uint32):
    return a.ctypes.data_as(ctypes.POINTER(ty))


# ---- points <-> limb arrays (Montgomery form, affine (x, y), infinity = all-zero) --------------
def fq_limbs(curve):
    return curve.fq_limbs64 * 2


def pack_points(curve, group, pts):
    """Affine oracle points (ints or Fq2 tuples, None = infinity) -> uint32 array in the C-ABI layout."""
    n = fq_limbs(curve)
    R = 1 << (32 * n)
    p = curve.p
    flat = []
    for P in pts:
        if P is None:
            flat += [0] * (2 * group)
        elif group == 1:
            flat += [P[0] * R % p, P[1] * R % p]
        else:
            flat += [P[0][0] * R % p, P[0][1] * R % p, P[1][0] * R % p, P[1][1] * R % p]
    return pack_u32(flat, n)


def unpack_points(curve, group, arr):
    n = fq_limbs(curve)
    Rinv = pow(1 << (32 * n), -1, curve.p)
    vals = [v * Rinv % curve.p for v in unpack_u32(arr, n)]
    out = []
    step = 2 * group
    for i in range(0, len(vals), step):
        c = vals[i : i + step]
        if all(v == 0 for v in c):
            out.append(None)
        elif group == 1:
            out.append((c[0], c[1]))
        else:
            out.append(((c[0], c[1]), (c[2], c[3])))
    return out


def pack_fr(curve, xs, mont=True):
    R = 1 << 256
    return pack_u32([(x * R % curve.r) if mont else x % curve.r for x in xs], 8)


def unpack_fr(curve, arr, mont=True):
    Rinv = pow(1 << 256, -1, curve.r)
    return [(v * Rinv % curve.r) if mont else v for v in unpack_u32(arr, 8)]


# ---- R1CS / proving-key marshalling (oracle objects -> C-ABI arrays) ----------------------------
def csr_from_rows(curve, matrix):
    """Oracle Matrix (rows of (coeff, col)) -> (row_ptr u64, col u32, coeff limbs u32) in Montgomery form."""
    row_ptr = np.zeros(len(matrix) + 1, dtype=np.uint64)
    cols, coeffs = [], []
    for i, row in enumerate(matrix):
        for c, col in row:
            cols.append(col)
            coeffs.append(c)
        row_ptr[i + 1] = len(cols)
    col = np.array(cols, dtype=np.uint32) if cols else np.zeros(0, dtype=np.uint32)
    co = pack_fr(curve, coeffs) if coeffs else np.zeros(0, dtype=np.uint32)
    return row_ptr, col, co


def make_pk_desc(curve, pk, keep):
    """Oracle ProvingKey -> snark_b200.lib.PkDesc (full key).  `keep` receives the numpy arrays so they
    outlive the descriptor."""
    from snark_b200.lib import PkDesc

    d = PkDesc()
    d.n_instance = pk.num_instance
    d.n_witness = len(pk.l_query)
    d.domain_size = pk.domain

    def put(name, group, pts):
        arr = pack_points(curve, group, pts)
        keep.append(arr)
        setattr(d, name, arr.ctypes.data)
        return len(pts)

    put("alpha_g1", 1, [pk.alpha_g1]); put("beta_g1", 1, [pk.beta_g1]); put("delta_g1", 1, [pk.delta_g1])
    put("beta_g2", 2, [pk.beta_g2]); put("delta_g2", 2, [pk.delta_g2])
    d.a_len = put("a_query", 1, pk.a_query)
    d.b1_len = put("b_g1_query", 1, pk.b_g1_query)
    d.b2_len = put("b_g2_query", 2, pk.b_g2_query)
    d.h_len = put("h_query", 1, pk.h_query)
    d.l_len = put("l_query", 1, pk.l_query)
    return d


def random_fr_limbs(rng, n, bits=254):
    """n random field elements as raw limbs (uint32[n*8]), uniform in [0, 2^bits) (< r for both curves)."""
    a = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
    top = bits - 224
    a[:, 7] &= np.uint32((1 << top) - 1)
    return a.reshape(-1)


def limbs_to_ints(arr, n=8):
    """uint32[count*n] -> list of Python ints (vectorised per limb)."""
    a = np.asarray(arr, dtype=np.uint32).reshape(-1, n).astype(object)
    acc = a[:, 0].copy()
    for j in range(1, n):
        acc = acc + (a[:, j] << (32 * j))
    return list(acc)


def pairing_verify_packed(curve, vk, n_instance, z_inst, proof_abc):
    """Groth16 verification with real pairings (oracle/pairing.py) on C-ABI arrays: `vk` as returned by
    Backend.groth16_setup (dict of uint32 arrays), z_inst the instance assignment INCLUDING the leading 1 (ints),
    proof_abc the three uint32 arrays of Backend.groth16_prove."""
    from oracle import pairing

    vk_pts = {
        "alpha_g1": unpack_points(curve, 1, vk["alpha_g1"])[0],
        "beta_g2": unpack_points(curve, 2, vk["beta_g2"])[0],
        "gamma_g2": unpack_points(curve, 2, vk["gamma_g2"])[0],
        "delta_g2": unpack_points(curve, 2, vk["delta_g2"])[0],
        "gamma_abc_g1": unpack_points(curve, 1, vk["gamma_abc_g1"])[:n_instance],
    }
    a, b, c = proof_abc
    proof = (unpack_points(curve, 1, a)[0], unpack_points(curve, 2, b)[0], unpack_points(curve, 1, c)[0])
    return pairing.groth16_verify(vk_pts, list(z_inst[1:]), proof, curve)


# ---- synthetic proving keys of known discrete logs (GPU tests at full size) ----------------------
KEY_QUERIES = (("a_query", "a_len", 1), ("b_g1_query", "b1_len", 1), ("b_g2_query", "b2_len", 2), ("h_query", "h_len", 1),
               ("l_query", "l_len", 1))


def known_log_key(be, curve, consts, n_inst, n_wit, domain, seed, qap=0):
    """A proving key whose points are k G for random k known to the caller, as bench.py builds it: the k are drawn on the GPU
    (torch generator seeded with `seed`, below 2^253 and below r), multiplied by the fixed-base kernel and uploaded from
    device memory.  consts = (alpha, beta, delta) as ints; the h query has domain - 1 points (libsnark) or domain (qap = 1,
    circom).  The b_g1 and b_g2 queries get independent logs, which the algebra allows.  Returns (pk handle, dl) with
    dl[query] the canonical uint32 limbs of its k."""
    import torch

    from snark_b200.lib import MEM_DEVICE, PkDesc

    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    top = (1 << (min(253, curve.r.bit_length() - 1) - 224)) - 1
    n_vars = n_inst + n_wit
    lens = {"a_query": n_vars, "b_g1_query": n_vars, "b_g2_query": n_vars, "h_query": domain if qap else domain - 1,
            "l_query": n_wit}

    def query(group, n):
        k = torch.randint(-(1 << 31), (1 << 31) - 1, (n, 8), dtype=torch.int32, device=dev, generator=gen)
        k[:, 7] &= top
        out = torch.empty(n * (be.g1_bytes if group == 1 else be.g2_bytes) // 4, dtype=torch.int32, device=dev)
        be.fixed_base(group, k, n, mont=False, out=out)
        be.sync()
        return out, k.cpu().numpy().view(np.uint32).reshape(-1)

    c1 = be.fixed_base(1, pack_fr(curve, consts, mont=False), 3, mont=False)
    c2 = be.fixed_base(2, pack_fr(curve, consts[1:], mont=False), 2, mont=False)
    g1w, g2w = be.g1_bytes // 4, be.g2_bytes // 4
    c1t = torch.from_numpy(c1.view(np.int32)).to(dev)
    c2t = torch.from_numpy(c2.view(np.int32)).to(dev)
    d = PkDesc()
    d.n_instance, d.n_witness, d.domain_size = n_inst, n_wit, domain
    d.alpha_g1, d.beta_g1, d.delta_g1 = c1t.data_ptr(), c1t.data_ptr() + 4 * g1w, c1t.data_ptr() + 8 * g1w
    d.beta_g2, d.delta_g2 = c2t.data_ptr(), c2t.data_ptr() + 4 * g2w
    keep, dl = [], {}
    for name, ln, group in KEY_QUERIES:
        t, k = query(group, lens[name])
        keep.append(t)
        dl[name] = k
        setattr(d, name, t.data_ptr())
        setattr(d, ln, lens[name])
    return be.pk_upload(d, mem=MEM_DEVICE, qap=qap), dl


def known_log_proof(be, curve, consts, dl, z_inst, z_wit, h, r, s):
    """The proof (A, B, C) as affine oracle points that a key of known_log_key gives for z = z_inst || z_wit (Montgomery
    limbs), the witness map's h (Montgomery limbs, as many as the h query has points) and ints r, s: the exponents by
    dot products in Fr on the CPU (C++ oracle), the points by the oracle's scalar multiplication of the generators."""
    from oracle import cnative
    from oracle.ec import groups

    rm = curve.r
    z_all = np.concatenate([z_inst, z_wit])

    def dot(name, scal_mont):
        # fr_dot(k, s~) = sum k_i s~_i R^-1 = sum k_i s_i: read back as a canonical value
        n = len(dl[name]) // 8
        return unpack_fr(curve, cnative.fr_dot(be.curve, dl[name], scal_mont, n), mont=False)[0]

    alpha, beta, delta = consts
    a_star = (alpha + dot("a_query", z_all) + r * delta) % rm
    b1_star = (beta + dot("b_g1_query", z_all) + s * delta) % rm
    b2_star = (beta + dot("b_g2_query", z_all) + s * delta) % rm
    c_star = (s * a_star + r * b1_star - r * s % rm * delta + dot("l_query", z_wit) + dot("h_query", h)) % rm
    G1, G2 = groups(curve)
    return G1.mul(G1.gen, a_star), G2.mul(G2.gen, b2_star), G1.mul(G1.gen, c_star)
