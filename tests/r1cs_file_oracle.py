"""Writer of circom's .r1cs files.  TEST INFRASTRUCTURE ONLY.

Restated from the iden3 r1cs binfile spec, circom's writer and ark-circom's R1CSFile reader -- see snark_b200/csrc/zkey.cu
for the layout.  Neither circom nor ark-circom is in the reference tree and no file written by circom exists here, so this
writer and the library's reader are checked for consistency with each other only: byte parity with circom is NOT pinned.

Matrices are taken as C-ABI CSR triples (row_ptr uint64, col uint32, Montgomery coefficient limbs uint32, as
tests/util.csr_from_rows returns them) and the constraint section is assembled with numpy, so synthetic circuits of 2^24
constraints are written without Python loops over the entries; coefficients are converted once per distinct value.
"""
import struct

import numpy as np

from tests.zkey_oracle import binfile, fr_rescale

N8 = 32
ENTRY_WORDS = 1 + N8 // 4   # u32 wire, then the coefficient


def header_section(curve, n_wires, n_pub_out, n_pub_in, n_prv_in, n_labels, n_constraints, prime=None):
    """section 1: n8, the prime, nWires, nPubOut, nPubIn, nPrvIn (u32), nLabels (u64), mConstraints (u32)"""
    p = curve.r if prime is None else prime
    return (struct.pack("<I", N8) + int(p).to_bytes(N8, "little")
            + struct.pack("<IIIIQI", n_wires, n_pub_out, n_pub_in, n_prv_in, n_labels, n_constraints))


def constraint_words(curve, csr, mont=True):
    """section 2 as uint32 words: per constraint, for A, B, C, the count and then (wire, canonical coefficient) per entry.
    mont=False: the coefficient limbs of csr are canonical already"""
    n = len(csr[0][0]) - 1
    rps = [np.asarray(m[0], dtype=np.int64) for m in csr]
    counts = [np.diff(rp) for rp in rps]
    start = 3 * np.arange(n, dtype=np.int64) + ENTRY_WORDS * (rps[0][:-1] + rps[1][:-1] + rps[2][:-1])
    total = 3 * n + ENTRY_WORDS * sum(int(rp[-1]) for rp in rps)
    words = np.zeros(total, dtype=np.uint32)
    at = start.copy()   # the count word of matrix k in each constraint
    for k, (rp, col, coeff) in enumerate(csr):
        words[at] = counts[k]
        nnz = int(rp[-1])
        if nnz:
            rows = np.repeat(np.arange(n, dtype=np.int64), counts[k])
            pos = at[rows] + 1 + ENTRY_WORDS * (np.arange(nnz, dtype=np.int64) - rps[k][rows])
            words[pos] = np.asarray(col, dtype=np.uint32)
            canon = (fr_rescale(curve, coeff, pow(1 << 256, -1, curve.r)) if mont else np.asarray(coeff, dtype=np.uint32)).reshape(-1, 8)
            for j in range(8):
                words[pos + 1 + j] = canon[:, j]
        at = at + 1 + ENTRY_WORDS * counts[k]
    return words


def r1cs_sections(curve, csr, n_pub_out, n_pub_in, n_prv_in, n_wires=None, n_labels=None, wire_map=True, mont=True):
    """[(type, bytes)] of an .r1cs in circom's order: header, constraints, and (wire_map) the wire -> label map"""
    n_rows = len(csr[0][0]) - 1
    if n_wires is None:
        n_wires = 1 + max([n_pub_out + n_pub_in + n_prv_in] + [int(np.max(m[1])) for m in csr if len(m[1])])
    n_labels = n_wires if n_labels is None else n_labels
    secs = [(1, header_section(curve, n_wires, n_pub_out, n_pub_in, n_prv_in, n_labels, n_rows)),
            (2, constraint_words(curve, csr, mont).tobytes())]
    if wire_map:
        secs.append((3, np.arange(n_wires, dtype=np.uint64).tobytes()))
    return secs


def write_r1cs(curve, csr, n_pub_out, n_pub_in, n_prv_in, n_wires=None, n_labels=None, wire_map=True, order="circom", path=None,
               mont=True):
    """An .r1cs of the matrices csr = [A, B, C] (CSR, Montgomery) over z = One, n_pub_out public outputs, n_pub_in public
    inputs, n_prv_in private inputs and the internal wires.  order="circom": sections 1, 2, 3; "shuffled": constraints first,
    the map before the header and an unknown section added.  With `path` the file is written there and the path is
    returned; otherwise the bytes.  mont=False: the coefficient limbs of csr are canonical already (no conversion)."""
    secs = r1cs_sections(curve, csr, n_pub_out, n_pub_in, n_prv_in, n_wires, n_labels, wire_map, mont)
    if order == "shuffled":
        secs = [secs[1]] + secs[2:] + [(77, b"unknown section"), secs[0]]
    else:
        assert order == "circom", order
    if path is None:
        return binfile(b"r1cs", 1, secs)
    with open(path, "wb") as f:   # not through binfile: the file is not assembled in memory a second time
        f.write(b"r1cs" + struct.pack("<II", 1, len(secs)))
        for t, body in secs:
            f.write(struct.pack("<IQ", t, len(body)))
            f.write(body)
    return path
