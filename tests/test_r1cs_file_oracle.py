"""CPU: the test-side .r1cs writer (tests/r1cs_file_oracle.py) lays out a small circuit byte for byte as the iden3 r1cs
binfile spec describes it, so the GPU reader's tests rest on a writer that is checked by hand once."""
import struct

import numpy as np

from oracle.params import BN254
from tests import r1cs_file_oracle as ro
from tests.util import csr_from_rows


def test_writer_layout_by_hand():
    r = BN254.r
    # z = (One, out, in, prv, w4): constraint 0: (2 out + w4 + w4) * (in) = (r - 1) prv;  constraint 1: () * (One) = ()
    mats = [[[(2, 1), (1, 4), (1, 4)], []], [[(1, 2)], [(1, 0)]], [[(r - 1, 3)], []]]
    csr = [csr_from_rows(BN254, M) for M in mats]
    got = ro.write_r1cs(BN254, csr, 1, 1, 1, n_wires=5, n_labels=9)
    fe = lambda v: v.to_bytes(32, "little")
    entry = lambda w, v: struct.pack("<I", w) + fe(v)
    header = struct.pack("<I", 32) + fe(r) + struct.pack("<IIIIQI", 5, 1, 1, 1, 9, 2)
    c0 = (struct.pack("<I", 3) + entry(1, 2) + entry(4, 1) + entry(4, 1) + struct.pack("<I", 1) + entry(2, 1)
          + struct.pack("<I", 1) + entry(3, r - 1))
    c1 = struct.pack("<I", 0) + struct.pack("<I", 1) + entry(0, 1) + struct.pack("<I", 0)
    wire_map = np.arange(5, dtype=np.uint64).tobytes()
    want = b"r1cs" + struct.pack("<II", 1, 3)
    for t, body in ((1, header), (2, c0 + c1), (3, wire_map)):
        want += struct.pack("<IQ", t, len(body)) + body
    assert got == want
    assert len(header) == 32 + 32


def test_writer_to_a_path_equals_bytes(tmp_path):
    mats = [[[(1, 1)], [(3, 2), (4, 0)]], [[(1, 0)], []], [[(5, 2)], [(1, 1)]]]
    csr = [csr_from_rows(BN254, M) for M in mats]
    for order in ("circom", "shuffled"):
        data = ro.write_r1cs(BN254, csr, 0, 1, 0, order=order)
        path = ro.write_r1cs(BN254, csr, 0, 1, 0, order=order, path=tmp_path / "c.r1cs")
        assert path.read_bytes() == data
