"""Device-memory (mem = B2S_MEM_DEVICE) calls of b2s_spmv, b2s_witness_map(_qap) and b2s_witness_map_sim: the Backend
methods take host arrays only, so these call the C ABI with CUDA torch tensors and compare with the host results."""
import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests.util import csr_from_rows, pack_fr

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def test_device_buffers_equal_host_buffers(be):
    import torch

    from snark_b200 import lib as L

    curve = CURVES[be.curve]
    cs = orc.bench_circuit(curve, 200, seed=11)
    cs.finalize()
    mats, inst, wit = cs.to_matrices(), cs.instance_assignment, cs.witness_assignment
    n_rows = len(mats[0])
    m = be.r1cs_upload(n_rows, len(inst), len(wit), [csr_from_rows(curve, M) for M in mats])
    try:
        z = pack_fr(curve, list(inst) + list(wit))
        zd = torch.from_numpy(z.view(np.int32)).cuda()
        n_h = be.domain_size(m) * 8
        dev = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")
        host = lambda t: t.cpu().numpy().view(np.uint32)

        outs = [dev(n_rows * 8) for _ in range(3)]
        be._ck(be.lib.b2s_spmv(be.h, m, zd.data_ptr(), L.MEM_DEVICE, *[o.data_ptr() for o in outs]))
        be.sync()
        for got, want in zip(outs, be.spmv(m, z, n_rows)):
            assert np.array_equal(host(got), want)

        for qap in (L.QAP_LIBSNARK, L.QAP_CIRCOM):
            h = dev(n_h)
            be._ck(be.lib.b2s_witness_map_qap(be.h, m, zd.data_ptr(), L.MEM_DEVICE, qap, h.data_ptr()))
            be.sync()
            assert np.array_equal(host(h), be.witness_map(m, z, qap=qap)), qap

        h = dev(n_h)
        be._ck(be.lib.b2s_witness_map(be.h, m, zd.data_ptr(), L.MEM_DEVICE, h.data_ptr()))
        be.sync()
        assert np.array_equal(host(h), be.witness_map(m, z))

        h = dev(n_h)
        be._ck(be.lib.b2s_witness_map_sim(be.h, m, zd.data_ptr(), L.MEM_DEVICE, 1, h.data_ptr()))
        be.sync()
        assert np.array_equal(host(h), be.witness_map_sim(m, z, 1))
    finally:
        be.r1cs_free(m)
