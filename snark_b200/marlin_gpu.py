"""Device vector backend of the universal-setup (Marlin-style) path: every method is one C-ABI call into
libb200snark.so on device-resident vectors (see snark_b200/marlin.py for the protocol and the split host / device).

Vectors are CUDA torch tensors of shape [n, 8] int32 words (Fr, Montgomery limbs -- the layout of include/b200snark.h); torch is
used for what the task allows it for: device memory, copies and views.  All torch work is queued on the library's own stream
(`b2s_stream`, wrapped as an ExternalStream), so allocation, padding and the kernels are ordered without host synchronisation;
only commitments, evaluations and challenges come back to the host.

There is no CPU substitute: without libb200snark.so or without an sm_90 GPU the constructor raises."""
import numpy as np

from . import lib as L
from .marlin import log2

# field parameters the host needs for scalar conversion and transcript encoding (checked against the library's own constants by
# tests/test_gpu_marlin.py through a Montgomery round trip on the device)
_PARAMS = {
    L.BLS12_381: dict(
        r=0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001,
        p=0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab,
        gen=7, two_adicity=32),
    L.BN254: dict(
        r=21888242871839275222246405745257275088548364400416034343698204186575808495617,
        p=21888242871839275222246405745257275088696311157297823662689037894645226208583,
        gen=5, two_adicity=28),
    L.BLS12_377: dict(
        r=0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001,
        p=0x01ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001,
        gen=22, two_adicity=47),
}


class GpuBackend:
    def __init__(self, curve=L.BN254, device=0):
        import torch

        self.torch = torch
        self.be = L.Backend(curve=curve, device=device)      # raises without the library / an sm_90 GPU
        self.lib = self.be.lib
        self.h = self.be.h
        prm = _PARAMS[curve]
        self.r, self.p = prm["r"], prm["p"]
        self.coset_gen = prm["gen"]
        self._two_adicity = prm["two_adicity"]
        self._root = pow(prm["gen"], (self.r - 1) >> self._two_adicity, self.r)
        self.fq_bytes = self.be.fq_bytes
        self.fq_limbs = self.fq_bytes // 4
        self.R_fr = pow(2, 256, self.r)
        self.Rinv_fr = pow(self.R_fr, -1, self.r)
        self.Rinv_fq = pow(pow(2, 32 * self.fq_limbs, self.p), -1, self.p)
        self.dev = torch.device("cuda", device)
        self.stream = torch.cuda.ExternalStream(self.be.stream, device=self.dev)

    def close(self):
        self.be.close()

    @property
    def launches(self):
        return self.be.launches

    def omega(self, log_n):
        assert 0 <= log_n <= self._two_adicity
        return pow(self._root, 1 << (self._two_adicity - log_n), self.r)

    # ---- host <-> device -------------------------------------------------------------------------------------------------
    def _scalar(self, x):
        """One Montgomery Fr on the host (numpy uint32[8])."""
        v = (x % self.r) * self.R_fr % self.r
        return np.frombuffer(v.to_bytes(32, "little"), dtype=np.uint32).copy()

    def _ck(self, st):
        if st != 0:
            raise L.B2SError(st, self.lib.b2s_last_error(self.h).decode())

    def _new(self, n):
        with self.torch.cuda.stream(self.stream):
            return self.torch.empty((n, 8), dtype=self.torch.int32, device=self.dev)

    def from_ints(self, xs):
        buf = b"".join(((x % self.r) * self.R_fr % self.r).to_bytes(32, "little") for x in xs)
        host = self.torch.frombuffer(bytearray(buf), dtype=self.torch.int32).reshape(len(xs), 8)
        with self.torch.cuda.stream(self.stream):
            return host.to(self.dev)

    def to_ints(self, v):
        with self.torch.cuda.stream(self.stream):
            host = v.contiguous().cpu()
        self.be.sync()
        raw = host.numpy().tobytes()
        return [int.from_bytes(raw[32 * i: 32 * i + 32], "little") * self.Rinv_fr % self.r for i in range(len(v))]

    def pad(self, v, n):
        assert len(v) <= n
        with self.torch.cuda.stream(self.stream):
            out = self.torch.zeros((n, 8), dtype=self.torch.int32, device=self.dev)
            out[: len(v)].copy_(v)
        return out

    def slice(self, v, lo, hi):
        return v[lo:hi]                 # a view; rows are contiguous

    def concat(self, vs):
        with self.torch.cuda.stream(self.stream):
            return self.torch.cat(list(vs), dim=0)

    def shifted(self, v, sh):
        with self.torch.cuda.stream(self.stream):
            out = self.torch.zeros((sh + len(v), 8), dtype=self.torch.int32, device=self.dev)
            out[sh:].copy_(v)
        return out

    # ---- kernels ----------------------------------------------------------------------------------------------------------
    def _op(self, op, a, b=None, s=None, out=None):
        n = len(a)
        assert a.is_contiguous() and (b is None or (b.is_contiguous() and len(b) == n))
        out = self._new(n) if out is None else out
        sc = self._scalar(s) if s is not None else None
        self._ck(self.lib.b2s_poly_op(self.h, op, a.data_ptr(), b.data_ptr() if b is not None else None,
                                      sc.ctypes.data if sc is not None else None, out.data_ptr(), n, L.MEM_DEVICE))
        return out

    def mul(self, a, b):
        return self._op(0, a, b)

    def add(self, a, b):
        return self._op(1, a, b)

    def sub(self, a, b):
        return self._op(2, a, b)

    def scale(self, a, s):
        return self._op(3, a, s=s)

    def add_scalar(self, a, s):
        return self._op(4, a, s=s)

    def inv0(self, a):
        return self._op(5, a)

    def geom(self, n, c, s):
        out = self._new(n)
        cc, ss = self._scalar(c), self._scalar(s)
        self._ck(self.lib.b2s_poly_geom(self.h, cc.ctypes.data, ss.ctypes.data, n, L.MEM_DEVICE, out.data_ptr()))
        return out

    def eval(self, coeffs, z):
        assert coeffs.is_contiguous()
        zz = self._scalar(z)
        out = np.zeros(8, dtype=np.uint32)
        self._ck(self.lib.b2s_poly_eval(self.h, coeffs.data_ptr(), len(coeffs), zz.ctypes.data, L.MEM_DEVICE, out.ctypes.data))
        return int.from_bytes(out.tobytes(), "little") * self.Rinv_fr % self.r

    def ntt(self, v, inverse=False, coset=False):
        """Out of place (the protocol keeps its inputs): copy, then the in-place device transform."""
        assert v.is_contiguous()
        with self.torch.cuda.stream(self.stream):
            out = v.clone()
        self._ck(self.lib.b2s_ntt(self.h, out.data_ptr(), log2(len(out)), int(inverse), int(coset), L.MEM_DEVICE))
        return out

    # ---- matrices (CSR upload + SpMV of the Groth16 path, r1cs.cu) -----------------------------------------------------------
    def upload_matrices(self, mats, n_rows, n_cols):
        csr = []
        for M in mats:
            assert len(M) <= n_rows
            row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
            cols, coeffs = [], []
            for i in range(n_rows):
                if i < len(M):
                    for c, col in M[i]:
                        assert 0 <= col < n_cols
                        cols.append(col)
                        coeffs.append(((c % self.r) * self.R_fr % self.r).to_bytes(32, "little"))
                row_ptr[i + 1] = len(cols)
            csr.append((row_ptr, np.array(cols, dtype=np.uint32), np.frombuffer(b"".join(coeffs), dtype=np.uint32).copy()
                        if coeffs else np.zeros(0, dtype=np.uint32)))
        # z has n_cols entries: one "instance" column and n_cols - 1 "witness" columns as far as the handle is concerned
        return (self.be.r1cs_upload(n_rows, 1, n_cols - 1, csr), n_rows, n_cols)

    def spmv(self, handle, z, n):
        h, n_rows, n_cols = handle
        assert len(z) == n_cols and z.is_contiguous() and n_rows <= n
        with self.torch.cuda.stream(self.stream):
            outs = [self.torch.zeros((n, 8), dtype=self.torch.int32, device=self.dev) for _ in range(3)]
        self._ck(self.lib.b2s_spmv(self.h, h, z.data_ptr(), L.MEM_DEVICE, *[o.data_ptr() for o in outs]))
        return outs

    # ---- KZG10 -----------------------------------------------------------------------------------------------------------------
    def setup(self, size, tau):
        """`UniversalSetupSNARK::universal_setup` (snark/src/lib.rs:117-123): the powers tau^i G1, i < size, device resident.
        (The G2 half of the SRS -- tau H, two points -- is the verifier's; it is not needed to prove.)"""
        powers = self.geom(size, 1, tau)
        with self.torch.cuda.stream(self.stream):
            bases = self.torch.empty((size, self.be.g1_bytes // 4), dtype=self.torch.int32, device=self.dev)
        self._ck(self.lib.b2s_fixed_base_g1(self.h, powers.data_ptr(), size, 1, L.MEM_DEVICE, bases.data_ptr()))
        with self.torch.cuda.stream(self.stream):
            powers.zero_()               # tau's powers are toxic waste
        return bases

    def srs_size(self, srs):
        return len(srs)

    def commit(self, srs, coeffs, shift=0):
        n = len(coeffs)
        assert shift + n <= len(srs) and coeffs.is_contiguous()
        out = np.zeros(self.be.g1_bytes // 4, dtype=np.uint32)
        self._ck(self.lib.b2s_msm_g1(self.h, srs[shift:].data_ptr(), coeffs.data_ptr(), n, 1, L.MEM_DEVICE, out.ctypes.data))
        return self._point(out)

    def _point(self, limbs):
        raw = limbs.tobytes()
        x = int.from_bytes(raw[: self.fq_bytes], "little")
        y = int.from_bytes(raw[self.fq_bytes: 2 * self.fq_bytes], "little")
        if x == 0 and y == 0:
            return None
        return (x * self.Rinv_fq % self.p, y * self.Rinv_fq % self.p)
