"""Device Fp::inverse (divsteps) through b2s_field_op op 3 on all three curves, base and scalar field, at 2^16 random
elements plus the edge values of tests/test_host_inverse.py, against Python's pow(x, -1, p).  GPU only."""
import random

import numpy as np
import pytest

from oracle.params import BLS12_381, BN254
from tests import bls377_oracle as b7
from tests.test_host_inverse import edge_values
from tests.util import pack_u32, unpack_u32

pytestmark = pytest.mark.gpu
MODULI = {0: (BLS12_381.p, BLS12_381.r), 1: (BN254.p, BN254.r), 2: (b7.P, b7.R)}


@pytest.mark.parametrize("curve", [0, 1, 2], ids=["bls12_381", "bn254", "bls12_377"])
@pytest.mark.parametrize("field", [0, 1], ids=["fq", "fr"])
def test_inverse(curve, field):
    from snark_b200 import Backend

    be = Backend(curve=curve)
    try:
        p = MODULI[curve][field]
        n = (be.fq_bytes if field == 0 else be.fr_bytes) // 4
        R = 1 << (32 * n)
        Rinv = pow(R, -1, p)
        rng = random.Random(900 + 10 * curve + field)
        xs = edge_values(p, n) + [rng.randrange(p) for _ in range(1 << 16)]
        A = pack_u32(xs, n)
        got = unpack_u32(be.field_op(field, 3, A, np.zeros_like(A)), n)
        exp = [pow(x * Rinv % p, -1, p) * R % p if x else 0 for x in xs]
        bad = [i for i in range(len(xs)) if got[i] != exp[i]]
        assert not bad, (curve, field, len(bad), hex(xs[bad[0]]))
    finally:
        be.close()
