"""Groth16 under ark-circom's CircomReduction for the CPU oracle.  TEST INFRASTRUCTURE ONLY.

Restates `CircomReduction` (ark-circom's implementation of ark-groth16's `R1CSToQAP`, the reduction of snarkjs keys) from
its definition; neither ark-circom nor snarkjs is in the reference tree and no fixture of theirs can be produced offline, so
parity with their bytes is UNPINNED, as for the rest of oracle/groth16.py.  Everything but the witness map and the h query is
oracle/groth16.py's LibsnarkReduction key and prover, reused as is.

With N the domain size, w = omega_N and w2 = omega_2N (w2^2 = w), the odd coset is x_j = w2 w^j, where Z(x_j) = -2:
  witness map   a = A z (instance rows copied in), b = B z, c = a o b on H; a, b, c moved to the odd coset; h_j = a_j b_j - c_j
  h query       h_query[j] = L^(2N)_{2j+1}(tau) / delta G1, j < N   (odd-indexed Lagrange basis of the size-2N domain)
For a satisfying z, sum_j h_j L^(2N)_{2j+1}(tau) = H(tau) Z(tau) and h_j = -2 H(x_j) with H the libsnark quotient, so the
two reductions give the same proof for the same trapdoor, z, r and s.
"""
import dataclasses

from oracle import groth16 as og
from oracle.ec import groups
from oracle.msm import msm_pippenger
from oracle.ntt import coset_ntt, ntt
from oracle.r1cs import mat_vec_mul


def omega2(curve, N):
    """primitive 2N-th root of unity with omega2^2 = omega_N"""
    return curve.omega(N.bit_length())


def odd_coset_eval(curve, coeffs):
    """evaluations of the polynomial with these N coefficients at x_j = w2 w^j"""
    return coset_ntt(curve, coeffs, g=omega2(curve, len(coeffs)))


def witness_map_circom(curve, mats, z, num_instance):
    """CircomReduction::witness_map_from_matrices, steps 1-4 literally -> N odd-coset evaluations."""
    r = curve.r
    A, B, _C = mats                                         # C is never read
    n = len(A)
    N = og.domain_size(n, num_instance)
    a = mat_vec_mul(r, A, z) + [0] * (N - n)
    b = mat_vec_mul(r, B, z) + [0] * (N - n)
    for i in range(num_instance):
        a[n + i] = z[i]
    c = [x * y % r for x, y in zip(a, b)]
    a, b, c = (odd_coset_eval(curve, ntt(curve, v, inverse=True)) for v in (a, b, c))
    return [(a[j] * b[j] - c[j]) % r for j in range(N)]


def lagrange_odd_at_tau(curve, N, tau):
    """L^(2N)_{2j+1}(tau) = (tau^2N - 1) x / (2N (tau - x)), x = w2^(2j+1), j < N"""
    r = curve.r
    w2 = omega2(curve, N)
    zt2 = (pow(tau, 2 * N, r) - 1) % r
    assert zt2 != 0, "tau^(2N) = 1"
    scale = zt2 * pow(2 * N, -1, r) % r
    out, x, step = [], w2, w2 * w2 % r
    for _ in range(N):
        out.append(scale * x % r * pow((tau - x) % r, -1, r) % r)
        x = x * step % r
    return out


def setup_circom(curve, mats, num_instance, num_witness, td):
    """The libsnark key of oracle/groth16.py.setup with the circom h query (N points)."""
    pk = og.setup(curve, mats, num_instance, num_witness, td)
    G1 = groups(curve)[0]
    dinv = pow(td.delta, -1, curve.r)
    hq = [G1.mul(G1.gen, v * dinv % curve.r) for v in lagrange_odd_at_tau(curve, pk.domain, td.tau)]
    return dataclasses.replace(pk, h_query=hq)


def prove_circom(pk, mats, z_inst, z_wit, r_rand, s_rand, msm=msm_pippenger):
    """create_proof_with_reduction::<CircomReduction>: oracle/groth16.py's prover with the circom witness map.
    Returns affine (A, B, C) and h."""
    curve = pk.curve
    G1, G2 = groups(curve)
    z = list(z_inst) + list(z_wit)
    h = witness_map_circom(curve, mats, z, len(z_inst))
    J1 = G1.to_jac
    h_acc = J1(msm(G1, pk.h_query, h))
    l_acc = J1(msm(G1, pk.l_query, z_wit))

    def calc(G, query, vk_param, delta, rnd):
        acc = G.to_jac(msm(G, query[1:], z[1:]))
        res = G.jmul(G.to_jac(delta), rnd)
        res = G.jadd_affine(res, query[0])
        res = G.jadd(res, acc)
        return G.jadd_affine(res, vk_param)

    g_a = calc(G1, pk.a_query, pk.alpha_g1, pk.delta_g1, r_rand)
    g1_b = calc(G1, pk.b_g1_query, pk.beta_g1, pk.delta_g1, s_rand)
    g2_b = calc(G2, pk.b_g2_query, pk.beta_g2, pk.delta_g2, s_rand)
    rs = r_rand * s_rand % curve.r
    g_c = G1.jmul(g_a, s_rand)
    g_c = G1.jadd(g_c, G1.jmul(g1_b, r_rand))
    g_c = G1.jadd(g_c, G1.jneg(G1.jmul(G1.to_jac(pk.delta_g1), rs)))
    g_c = G1.jadd(g_c, l_acc)
    g_c = G1.jadd(g_c, h_acc)
    return G1.to_affine(g_a), G2.to_affine(g2_b), G1.to_affine(g_c), h


def expected_proof_exponents(pk, z_inst, z_wit, h, r_rand, s_rand):
    """Discrete logs (a*, b*, c*) of a circom proof under the known trapdoor: oracle/groth16.py's, with
    sum_j h_j L^(2N)_{2j+1}(tau) in place of H(tau) Z(tau)."""
    curve, td = pk.curve, pk.trapdoor
    r = curve.r
    z = list(z_inst) + list(z_wit)
    ell = len(z_inst)
    a_star = (td.alpha + sum(zj * aj for zj, aj in zip(z, pk.a_tau)) + r_rand * td.delta) % r
    b_star = (td.beta + sum(zj * bj for zj, bj in zip(z, pk.b_tau)) + s_rand * td.delta) % r
    dinv = pow(td.delta, -1, r)
    wit = sum(z[j] * (td.beta * pk.a_tau[j] + td.alpha * pk.b_tau[j] + pk.c_tau[j]) for j in range(ell, len(z))) % r
    hz = sum(hj * lj for hj, lj in zip(h, lagrange_odd_at_tau(curve, pk.domain, td.tau))) % r
    c_star = ((wit + hz) * dinv + s_rand * a_star + r_rand * b_star - r_rand * s_rand % r * td.delta) % r
    return a_star, b_star, c_star


def check_in_exponent(pk, proof, z_inst, z_wit, h, r_rand, s_rand):
    """True iff proof == (a* G1, b* G2, c* G1) for the circom exponents."""
    G1, G2 = groups(pk.curve)
    a_star, b_star, c_star = expected_proof_exponents(pk, z_inst, z_wit, h, r_rand, s_rand)
    A, B, C = proof[:3]
    return A == G1.mul(G1.gen, a_star) and B == G2.mul(G2.gen, b_star) and C == G1.mul(G1.gen, c_star)
