#!/usr/bin/env python3
"""Time of loading a circom .r1cs onto the GPU against the ark-circom-like route, one run.

For each --log-n: builds a synthetic circom-shaped R1CS of 2^log_n - 4 constraints (3 public signals; per constraint A holds
1-3 entries, B 1, C 1-2, coefficients mostly 1, some -1 and a few other values) on --curve, writes it with the test-side
writer (tests/r1cs_file_oracle.py) to a temporary file, maps it with np.memmap and times, with the host clock around
synchronising calls (after one warm-up of every step at 2^12):
  - b2s_r1cs_file_load; and, reported separately, the host walk of the count words: the same call on the file with
    mConstraints lowered by one, which walks every count word, stops at "bytes after its constraints" and allocates nothing;
  - the ark-circom-like route to the same handle: the file parsed to CSR on the host (a Python walk of the count words, as
    R1CSFile reads them one by one, then numpy for the entries) plus b2s_r1cs_upload (host-side coefficient interning);
  - b2s_witness_map on both handles (z and h on the device), alternating, --reps times each (median, min and max).
It checks that both handles give the same witness-map output bits.  Prints one JSON line per --log-n with the card name and
power limit read in the same run.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_PUB_OUT, N_PUB_IN, N_PRV_IN = 1, 2, 2
M_CONSTRAINTS_AT = 12 + 12 + 4 + 32 + 16 + 8   # byte of mConstraints when the header is the first section


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return "unknown", "unknown"


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, round(time.perf_counter() - t0, 4)


def synthetic(curve, log_n, seed):
    """(n_rows, n_wires, csr with Montgomery coefficients, the same with canonical ones)"""
    from tests.util import pack_fr

    rng = np.random.default_rng(seed)
    n_inst = 1 + N_PUB_OUT + N_PUB_IN
    n_rows = (1 << log_n) - n_inst
    n_wires = n_rows + n_inst + N_PRV_IN
    vals = [1, curve.r - 1, 2, 3, (curve.r + 1) // 2]
    mont = pack_fr(curve, vals).reshape(-1, 8)
    canon = pack_fr(curve, vals, mont=False).reshape(-1, 8)
    csr_m, csr_c = [], []
    for lo, hi in ((1, 3), (1, 1), (1, 2)):
        counts = rng.integers(lo, hi + 1, size=n_rows)
        row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
        row_ptr[1:] = np.cumsum(counts)
        nnz = int(row_ptr[-1])
        col = rng.integers(0, n_wires, size=nnz, dtype=np.uint32)
        pick = rng.choice(len(vals), size=nnz, p=[0.85, 0.1, 0.02, 0.02, 0.01])
        csr_m.append((row_ptr, col, mont[pick].reshape(-1)))
        csr_c.append((row_ptr, col, canon[pick].reshape(-1)))
    return n_rows, n_wires, csr_m, csr_c


def parse_to_csr(curve, data):
    """the ark-circom-like host parse: framing, then the count words one by one, then the entries with numpy -> CSR with
    Montgomery coefficients (n_rows, n_instance, n_witness, csr)"""
    from tests.zkey_oracle import fr_rescale

    buf = np.asarray(data).view(np.uint8)
    n_sec, at, sec = int(buf[8:12].view(np.uint32)[0]), 12, {}
    for _ in range(n_sec):
        t, size = int(buf[at: at + 4].view(np.uint32)[0]), int(buf[at + 4: at + 12].view(np.uint64)[0])
        sec[t] = (at + 12, size)
        at += 12 + size
    h = buf[sec[1][0]: sec[1][0] + sec[1][1]]
    n8 = int(h[:4].view(np.uint32)[0])
    n_wires, n_out, n_in, _n_prv = (int(x) for x in h[4 + n8: 20 + n8].view(np.uint32))
    m = int(h[28 + n8: 32 + n8].view(np.uint32)[0])
    off, size = sec[2]
    words = buf[off: off + size].view(np.uint32)
    w, flat, p = memoryview(words), [0] * (3 * m), 0
    for t in range(3 * m):   # the sequential part: each count word's position depends on every count before it
        c = w[p]
        flat[t] = c
        p += 1 + 9 * c
    counts = np.array(flat, dtype=np.int64).reshape(m, 3).T
    starts = 3 * np.arange(m, dtype=np.int64) + 9 * (np.cumsum(counts.sum(axis=0)) - counts.sum(axis=0))
    csr, at = [], starts.copy()
    for k in range(3):
        row_ptr = np.zeros(m + 1, dtype=np.uint64)
        row_ptr[1:] = np.cumsum(counts[k])
        nnz = int(row_ptr[-1])
        rows = np.repeat(np.arange(m, dtype=np.int64), counts[k])
        pos = at[rows] + 1 + 9 * (np.arange(nnz, dtype=np.int64) - row_ptr[:-1].astype(np.int64)[rows])
        col = words[pos]
        canon = np.stack([words[pos + 1 + j] for j in range(8)], axis=1)
        uniq, inv = np.unique(canon.view(np.dtype((np.void, 32))).reshape(-1), return_inverse=True)   # converted once per value
        mont = fr_rescale(curve, uniq.view(np.uint32), 1 << 256).reshape(-1, 8)
        csr.append((row_ptr, np.ascontiguousarray(col), np.ascontiguousarray(mont[np.asarray(inv).reshape(-1)]).reshape(-1)))
        at = at + 1 + 9 * counts[k]
    n_inst = 1 + n_out + n_in
    return m, n_inst, n_wires - n_inst, csr


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--log-n", type=int, nargs="+", default=[16, 20, 24])
    ap.add_argument("--curve", choices=["bls12_381", "bn254", "bls12_377"], default="bn254")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch

    from oracle.params import BLS12_381, BN254
    from snark_b200 import B2SError, Backend
    from snark_b200.lib import MEM_DEVICE
    from tests import r1cs_file_oracle as ro
    from tests.bls377_oracle import BLS12_377
    from tests.util import pack_fr

    curve_id = {"bls12_381": 0, "bn254": 1, "bls12_377": 2}[a.curve]
    curve = [BLS12_381, BN254, BLS12_377][curve_id]
    be = Backend(curve=curve_id)
    name, power = card()
    tmp = tempfile.mkdtemp(prefix="r1cs_probe_")

    def run(log_n, reps):
        n_rows, n_wires, csr_m, csr_c = synthetic(curve, log_n, seed=log_n)
        path = os.path.join(tmp, f"synthetic_{log_n}.r1cs")
        ro.write_r1cs(curve, csr_c, N_PUB_OUT, N_PUB_IN, N_PRV_IN, n_wires=n_wires, path=path, mont=False)
        del csr_c
        data = np.memmap(path, dtype=np.uint8, mode="r+")
        nnz = [int(c[0][-1]) for c in csr_m]
        res = {"log_n": log_n, "constraints": n_rows, "nnz": nnz, "file_bytes": int(data.nbytes)}
        m_file, res["file_load_s"] = timed(lambda: (be.r1cs_file_load(data), be.sync())[0])
        # the walk alone: one constraint fewer in the header, so the walk ends with bytes left and the load stops there
        data[M_CONSTRAINTS_AT: M_CONSTRAINTS_AT + 4] = np.frombuffer(np.uint32(n_rows - 1).tobytes(), dtype=np.uint8)
        t0 = time.perf_counter()
        try:
            be.r1cs_file_load(data)
            raise AssertionError("the shortened header was accepted")
        except B2SError as e:
            assert "bytes after its" in str(e), str(e)
        res["host_walk_s"] = round(time.perf_counter() - t0, 4)
        data[M_CONSTRAINTS_AT: M_CONSTRAINTS_AT + 4] = np.frombuffer(np.uint32(n_rows).tobytes(), dtype=np.uint8)

        def ark_route():
            m, n_inst, n_wit, csr = parse_to_csr(curve, data)
            t_parse = time.perf_counter() - t0
            h = be.r1cs_upload(m, n_inst, n_wit, csr)
            be.sync()
            return h, t_parse

        t0 = time.perf_counter()
        m_up, t_parse = ark_route()
        res["ark_route_s"] = round(time.perf_counter() - t0, 4)
        res["ark_parse_s"] = round(t_parse, 4)
        res["ark_upload_s"] = round(res["ark_route_s"] - t_parse, 4)
        res["load_speedup"] = round(res["ark_route_s"] / res["file_load_s"], 2)
        z = pack_fr(curve, [1] + [random.Random(log_n).randrange(curve.r) for _ in range(min(n_wires, 1 << 12) - 1)])
        z = np.resize(z, n_wires * 8)   # a full-width assignment from a few thousand distinct values
        zt = torch.from_numpy(z.view(np.int32)).cuda()
        hs = {key: torch.zeros(be.domain_size(m_file) * 8, dtype=torch.int32, device="cuda") for key in ("file", "upload")}
        torch.cuda.synchronize()

        def wmap(h, key):   # device z and h: the time is the witness map, not the copies
            be._ck(be.lib.b2s_witness_map(be.h, h, zt.data_ptr(), MEM_DEVICE, hs[key].data_ptr()))
            be.sync()

        for key, h in (("file", m_file), ("upload", m_up)):
            wmap(h, key)   # warm-up of this shape
        res["witness_map_equal"] = bool(torch.equal(hs["file"], hs["upload"]))
        times = {"file": [], "upload": []}
        for _ in range(reps):
            for key, h in (("file", m_file), ("upload", m_up)):
                _, dt = timed(lambda: wmap(h, key))
                times[key].append(dt)
        for key, ts in times.items():
            res[f"witness_map_{key}_s"] = {"median": float(np.median(ts)), "min": min(ts), "max": max(ts)}
        be.r1cs_free(m_file)
        be.r1cs_free(m_up)
        del data
        os.remove(path)
        return res

    run(12, 1)   # warm-up: kernels, pinned buffers, NTT plans
    for log_n in a.log_n:
        out = {"tool": "r1cs_probe", "curve": a.curve, "gpu": name, "power_limit": power}
        out.update(run(log_n, a.reps))
        print(json.dumps(out), flush=True)
    os.rmdir(tmp)
    be.close()


if __name__ == "__main__":
    main()
