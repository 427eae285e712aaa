#!/usr/bin/env python3
"""Batched Groth16 verification throughput (b2s_groth16_verify_batch) on one GPU.

    python tools/verify_bench.py --curve bls12_381 --log-n 20 --n-inputs 16 --mem host

Proofs are simulated (a verifying key with known logs, c = (ab - alpha beta - gamma IC) / delta), 2^12 distinct ones tiled
to 2^log_n: the work per proof does not depend on its values.  One proof in 64 of the distinct set is broken (A + G1) and
every verdict is checked.  Prints one JSON line: proofs/s over the timed calls, the per-kernel split from a separate profiled
call, the time outside the kernels (host copies), the card and its power limit, and the algorithmic Fq-multiplication count
per verification with that count times proofs/s as a fraction of the 2.6e10 Fq mul/s ceiling of DESIGN.md section 4 (that
ceiling is the 381-bit one; for BN254 the fraction is against the same figure).

With --rlc the same batch, all valid, goes through groth16_verify_all (b2s_groth16_verify_batch_rlc, one verdict per
batch) and groth16_verify_batch in alternation; the line reports both rates, their ratio, both kernel splits and the
operation counts of both paths, and the batch with the broken proofs must be rejected.

With --bytes the batch is serialized (compressed ark Proofs, a || b || c) and goes through groth16_verify_batch_bytes
(with --rlc: groth16_verify_all_bytes) in alternation with two alternatives on the same proofs: the points path on
already-decoded points, and what a caller without the bytes path does -- split the bytes into three arrays, three validated
deserialize_points calls, then the points path.  The line reports the three rates, the bytes path's kernel split with the
decode kernels' share, and the decode operation count; a batch with malformed and invalid proofs must get the expected
verdicts and reasons."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import gen_field_params as gp  # noqa: E402  (loop constants)

CEILING = 2.6e10


def fq_mul_count(curve, n_inputs):
    """Fq multiplications of one verification, from the loop constants and the operation counts of pairing.cuh
    (Fq2 mul 3, Fq2 square 2, Fq2 x Fq 2; Fq inverse ~ bits + bits / 2)."""
    bls = curve == "bls12_381"
    bits = 381 if bls else 254
    inv_fq = bits + bits // 2
    digits = [int(b) for b in bin(gp.BLS_X_ABS)[2:]] if bls else gp.naf(6 * gp.BN_X + 2)
    steps, adds = len(digits) - 1, sum(1 for d in digits[1:] if d)
    sqr12, mul12, cyc, ell, dbl, add = 36, 54, 18, 43, 28, 37
    miller = (steps - 1) * sqr12 + steps * (dbl + 3 * ell) + adds * (add + 3 * ell)
    if not bls:
        miller += 2 * (6 + add + ell) + 2 * 2 * ell      # pi(Q), -pi^2(Q) lines: on the fly for B, prepared for the other two
    inv12 = 36 + 15 + 9 + (4 + inv_fq + 2) + 9 + 36
    xabs = gp.BLS_X_ABS if bls else gp.BN_X
    exp_x = (xabs.bit_length() - 1) * cyc + (bin(xabs).count("1") - 1) * mul12
    easy = inv12 + 2 * mul12 + 10
    hard = (5 * exp_x + 5 * mul12 + 15 + 10 + cyc) if bls else (3 * exp_x + 3 * cyc + 9 * mul12 + 15 + 10 + 15)
    ic = n_inputs * 32 * 255 / 256 * 10 + inv_fq + 3
    return int(miller + easy + hard + ic)


def fq_mul_count_rlc(curve, nf=2, log_n=20):
    """Fq multiplications per proof of the random-linear-combination check (b2s_groth16_verify_batch_rlc), the same
    operation counts as fq_mul_count: a one-pair Miller loop with B's lines on the fly whose Fq12 squarings are shared by nf
    proofs, rho A by 128-bit double-and-add in XYZZ (dbl 10, add 14) with one inversion, the share of the C MSM (signed
    windows of c bits over the 255-bit scalar, one mixed XYZZ addition of 10 per point and window) and of the product of
    the Miller values.  The per-batch terms (one final exponentiation, two prepared pairs, e(alpha, beta)^S, IC*) are
    left out: they are shared by 2^log_n proofs.  The public-input sums cost Fr multiplications, not counted."""
    bls = curve == "bls12_381"
    bits = 381 if bls else 254
    inv_fq = bits + bits // 2
    digits = [int(b) for b in bin(gp.BLS_X_ABS)[2:]] if bls else gp.naf(6 * gp.BN_X + 2)
    steps, adds = len(digits) - 1, sum(1 for d in digits[1:] if d)
    sqr12, mul12, ell, dbl, add = 36, 54, 43, 28, 37
    miller = (steps - 1) * sqr12 / nf + steps * (dbl + ell) + adds * (add + ell)
    if not bls:
        miller += 2 * (6 + add + ell)
    scalar = 127 * 10 + 64 * 14 + inv_fq + 3
    c = max(8, log_n - 4)
    msm = (255 // c + 1) * 10
    product = mul12 / nf
    return int(miller + scalar + msm + product)


def fq_mul_count_decode(curve):
    """Fq multiplications of decoding one compressed proof with validation (verify_decode_g1 / _g2): the square roots are
    powers to (p - 3) / 4 (bits - 1 squarings and popcount - 1 multiplications; the Fq2 root by the norm method takes one
    for the norm and on average 1.5 for delta), the subgroup criteria are scalar multiplications by the endomorphism scalar
    in XYZZ (dbl 10, add 14; x3 over Fq2): [|x|] twice per BLS12-381 G1 point, [|x|] / [6 x^2] once per G2 point, none for
    BN254 G1 (cofactor 1).  Montgomery conversions and comparisons are left out."""
    bls = curve == "bls12_381"
    p = gp.BLS_P if bls else gp.BN_P
    e = (p - 3) // 4
    pw = (e.bit_length() - 1) + (bin(e).count("1") - 1)
    k = gp.BLS_X_ABS if bls else 6 * gp.BN_X * gp.BN_X
    smul = (k.bit_length() - 1) * 10 + (bin(k).count("1") - 1) * 14
    g1 = pw + 4 + (2 * smul if bls else 0)
    g2 = 2.5 * pw + 3 * 8 + 3 * smul
    return int(2 * g1 + g2)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", choices=["bls12_381", "bn254"], default="bls12_381")
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--n-inputs", type=int, default=1)
    ap.add_argument("--mem", choices=["host", "device"], default="host")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rlc", action="store_true", help="time groth16_verify_all (one verdict per batch) against the per-proof path")
    ap.add_argument("--bytes", action="store_true", help="time the serialized-proof path against decoded points and decode-to-host")
    args = ap.parse_args()
    if args.bytes:
        return main_bytes(args)
    if args.rlc:
        return main_rlc(args)

    from snark_b200 import Backend
    from tests.test_gpu_verify import Sim

    be = Backend(curve=0 if args.curve == "bls12_381" else 1)
    rng = random.Random(20)
    sim = Sim(be, rng, args.n_inputs)
    base = 1 << min(12, args.log_n)
    x, a, b = sim.scalars(rng, base)
    c = sim.c_of(x, a, b)
    broken = set(range(0, base, 64))
    a = [(v + 1) % sim.curve.r if i in broken else v for i, v in enumerate(a)]
    inputs, A, B, C = sim.arrays(x, a, b, c)
    n = 1 << args.log_n
    reps = n // base
    inputs = np.tile(inputs, reps) if inputs is not None else None
    A, B, C = np.tile(A, reps), np.tile(B, reps), np.tile(C, reps)
    want = np.tile(np.array([i not in broken for i in range(base)]), reps)
    if args.mem == "device":
        import torch

        dev = torch.device("cuda")
        t = lambda arr: torch.from_numpy(arr.view(np.int32)).to(dev)
        inputs = t(inputs) if inputs is not None else None
        A, B, C = t(A), t(B), t(C)
        okd = torch.zeros(n, dtype=torch.uint8, device=dev)

        def run():
            be.groth16_verify_batch(sim.pvk, inputs, args.n_inputs, A, B, C, n_proofs=n, ok=okd)
            be.sync()
            return okd.cpu().numpy().astype(bool)
    else:
        def run():
            return be.groth16_verify_batch(sim.pvk, inputs, args.n_inputs, A, B, C)

    assert np.array_equal(run(), want), "verdicts differ from the expected ones"   # warm-up, and the check
    times = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        ok = run()
        times.append(time.perf_counter() - t0)
        assert np.array_equal(ok, want)
    be.profile(True)
    t0 = time.perf_counter()
    run()
    prof_s = time.perf_counter() - t0
    rep = be.profile_report()
    be.profile(False)
    kern = {k: round(v[1], 3) for k, v in rep.items()}
    best = min(times)
    pps = n / best
    muls = fq_mul_count(args.curve, args.n_inputs)
    name, power = gpu_info()
    print(json.dumps({
        "curve": args.curve, "n_proofs": n, "n_inputs": args.n_inputs, "mem": args.mem,
        "seconds": [round(s, 4) for s in times], "proofs_per_s": round(pps, 1),
        "kernel_ms": kern, "outside_kernels_ms": round(prof_s * 1e3 - sum(kern.values()), 3),
        "fq_mul_per_verification": muls, "fq_mul_per_s": round(muls * pps, 1), "fraction_of_ceiling": round(muls * pps / CEILING, 4),
        "gpu": name, "power_limit": power, "invalid_checked": int((~want).sum()),
    }))
    be.pvk_free(sim.pvk)
    be.close()


def main_rlc(args):
    """The same tiled batch, all valid, through groth16_verify_all and groth16_verify_batch in alternation; then the batch
    with one proof in 64 broken must give False.  rho is drawn once per batch outside the timed calls."""
    from snark_b200 import Backend
    from snark_b200.lib import random_rho
    from tests.test_gpu_verify import Sim

    be = Backend(curve=0 if args.curve == "bls12_381" else 1)
    rng = random.Random(20)
    sim = Sim(be, rng, args.n_inputs)
    base = 1 << min(12, args.log_n)
    x, a, b = sim.scalars(rng, base)
    c = sim.c_of(x, a, b)
    broken = set(range(0, base, 64))
    a_bad = [(v + 1) % sim.curve.r if i in broken else v for i, v in enumerate(a)]
    n = 1 << args.log_n
    reps = n // base
    tile = lambda arrs: [np.tile(v, reps) if v is not None else None for v in arrs]
    inputs, A, B, C = tile(sim.arrays(x, a, b, c))
    A_bad = tile(sim.arrays(x, a_bad, b, c))[1]
    if args.mem == "device":
        import torch

        dev = torch.device("cuda")
        t = lambda arr: torch.from_numpy(arr.view(np.int32)).to(dev) if arr is not None else None
        inputs, A, B, C, A_bad = t(inputs), t(A), t(B), t(C), t(A_bad)
        rho = t(random_rho(n))
        okd = torch.zeros(n, dtype=torch.uint8, device=dev)

        def per_proof():
            be.groth16_verify_batch(sim.pvk, inputs, args.n_inputs, A, B, C, n_proofs=n, ok=okd)
            be.sync()
            return bool(okd.all().item())
    else:
        rho = random_rho(n)

        def per_proof():
            return bool(be.groth16_verify_batch(sim.pvk, inputs, args.n_inputs, A, B, C).all())

    rlc = lambda a_: be.groth16_verify_all(sim.pvk, inputs, args.n_inputs, a_, B, C, rho=rho, n_proofs=n)
    assert rlc(A) and per_proof(), "an all-valid batch must be accepted"     # warm-up, and the checks
    assert not rlc(A_bad), "a batch with broken proofs must be rejected"
    t_rlc, t_pp = [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        assert rlc(A)
        t_rlc.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        assert per_proof()
        t_pp.append(time.perf_counter() - t0)
    split = {}
    for name, fn in (("rlc", lambda: rlc(A)), ("per_proof", per_proof)):
        be.profile(True)
        t0 = time.perf_counter()
        fn()
        prof_s = time.perf_counter() - t0
        rep = be.profile_report()
        be.profile(False)
        kern = {k: round(v[1], 3) for k, v in rep.items()}
        split[name] = {"kernel_ms": kern, "outside_kernels_ms": round(prof_s * 1e3 - sum(kern.values()), 3)}
    pps_rlc, pps_pp = n / min(t_rlc), n / min(t_pp)
    muls_rlc, muls_pp = fq_mul_count_rlc(args.curve, log_n=args.log_n), fq_mul_count(args.curve, args.n_inputs)
    name, power = gpu_info()
    print(json.dumps({
        "curve": args.curve, "n_proofs": n, "n_inputs": args.n_inputs, "mem": args.mem,
        "rlc_seconds": [round(s, 4) for s in t_rlc], "per_proof_seconds": [round(s, 4) for s in t_pp],
        "rlc_proofs_per_s": round(pps_rlc, 1), "per_proof_proofs_per_s": round(pps_pp, 1), "ratio": round(pps_rlc / pps_pp, 3),
        "split": split, "fq_mul_per_proof_rlc": muls_rlc, "fq_mul_per_proof": muls_pp,
        "count_ratio": round(muls_pp / muls_rlc, 3), "gpu": name, "power_limit": power, "invalid_rejected": len(broken) * reps,
    }))
    be.pvk_free(sim.pvk)
    be.close()


def main_bytes(args):
    """One tiled batch of compressed proofs, all valid, through the bytes path, the points path on the decoded points and the
    decode-to-host workflow in alternation (per proof, or with --rlc one verdict per batch); then a batch with one proof in
    64 algebraically broken (A + G1) and one in 64 malformed (C's flag bit) must get the expected verdicts and reasons."""
    from snark_b200 import Backend
    from snark_b200.lib import random_rho
    from tests.test_gpu_verify import Sim

    if args.mem != "host":
        raise SystemExit("--bytes times host batches")
    be = Backend(curve=0 if args.curve == "bls12_381" else 1)
    rng = random.Random(20)
    sim = Sim(be, rng, args.n_inputs)
    ni = args.n_inputs
    base = 1 << min(12, args.log_n)
    x, a, b = sim.scalars(rng, base)
    c = sim.c_of(x, a, b)
    n = 1 << args.log_n
    reps = n // base
    g1e, g2e = be.fq_bytes, 2 * be.fq_bytes   # compressed encodings

    def encode(A_, B_, C_):
        parts = [np.frombuffer(be.serialize_points(g, arr, base, True), dtype=np.uint8).reshape(base, -1)
                 for g, arr in ((1, A_), (2, B_), (1, C_))]
        return np.concatenate(parts, axis=1)

    inputs, A0, B0, C0 = sim.arrays(x, a, b, c)
    blob = np.tile(encode(A0, B0, C0), (reps, 1)).reshape(-1)
    inputs = np.tile(inputs, reps) if inputs is not None else None
    A, B, C = np.tile(A0, reps), np.tile(B0, reps), np.tile(C0, reps)
    # the check batch: A + G1 at i = 0 mod 64, C's flag bit flipped at i = 32 mod 64
    broken, malformed = set(range(0, base, 64)), set(range(32, base, 64))
    A_bad = sim.arrays(x, [(v + 1) % sim.curve.r if i in broken else v for i, v in enumerate(a)], b, c)[1]
    bad = encode(A_bad, B0, C0)
    flag = (g1e + g2e) + (0 if be.curve == 0 else g1e - 1)
    for i in malformed:
        bad[i, flag] ^= 0x80 if be.curve == 0 else 0x40
    bad = np.tile(bad, (reps, 1)).reshape(-1)
    want_ok = np.tile(np.array([i not in broken and i not in malformed for i in range(base)]), reps)
    want_reason = np.tile(np.array([48 + 1 if i in malformed else 0 for i in range(base)], dtype=np.uint8), reps)
    rho = random_rho(n)

    def split(data):   # what a caller does first without the bytes path: three contiguous arrays of encodings
        rows = data.reshape(n, -1)
        return rows[:, :g1e].copy(), rows[:, g1e:g1e + g2e].copy(), rows[:, g1e + g2e:].copy()

    def decode_host(data):
        ea, eb, ec = split(data)
        return (be.deserialize_points(1, ea, n, True, True), be.deserialize_points(2, eb, n, True, True),
                be.deserialize_points(1, ec, n, True, True))

    if args.rlc:
        paths = {
            "bytes": lambda: be.groth16_verify_all_bytes(sim.pvk, inputs, ni, blob, rho=rho)[0],
            "points": lambda: be.groth16_verify_all(sim.pvk, inputs, ni, A, B, C, rho=rho),
            "decode_host": lambda: be.groth16_verify_all(sim.pvk, inputs, ni, *decode_host(blob), rho=rho),
        }
        verdict, reason = be.groth16_verify_all_bytes(sim.pvk, inputs, ni, bad, rho=rho)
        assert not verdict and np.array_equal(reason, want_reason), "the batch with broken proofs must be rejected"
    else:
        paths = {
            "bytes": lambda: bool(be.groth16_verify_batch_bytes(sim.pvk, inputs, ni, blob)[0].all()),
            "points": lambda: bool(be.groth16_verify_batch(sim.pvk, inputs, ni, A, B, C).all()),
            "decode_host": lambda: bool(be.groth16_verify_batch(sim.pvk, inputs, ni, *decode_host(blob)).all()),
        }
        ok, reason = be.groth16_verify_batch_bytes(sim.pvk, inputs, ni, bad)
        assert np.array_equal(ok, want_ok) and np.array_equal(reason, want_reason), "verdicts differ from the expected ones"
    for name, fn in paths.items():
        assert fn(), name   # warm-up, and the all-valid check
    times = {name: [] for name in paths}
    for _ in range(args.steps):
        for name, fn in paths.items():
            t0 = time.perf_counter()
            assert fn(), name
            times[name].append(time.perf_counter() - t0)
    be.profile(True)
    t0 = time.perf_counter()
    paths["bytes"]()
    prof_s = time.perf_counter() - t0
    rep = be.profile_report()
    be.profile(False)
    kern = {k: round(v[1], 3) for k, v in rep.items()}
    decode_ms = sum(v for k, v in kern.items() if k.startswith("verify_decode"))
    pps = {name: n / min(t) for name, t in times.items()}
    muls_dec = fq_mul_count_decode(args.curve)
    muls_ver = fq_mul_count_rlc(args.curve, log_n=args.log_n) if args.rlc else fq_mul_count(args.curve, ni)
    name, power = gpu_info()
    print(json.dumps({
        "curve": args.curve, "n_proofs": n, "n_inputs": ni, "mem": "host", "mode": "rlc" if args.rlc else "per_proof",
        "seconds": {k: [round(s, 4) for s in v] for k, v in times.items()},
        "proofs_per_s": {k: round(v, 1) for k, v in pps.items()},
        "bytes_vs_points": round(pps["bytes"] / pps["points"], 3), "bytes_vs_decode_host": round(pps["bytes"] / pps["decode_host"], 3),
        "kernel_ms": kern, "decode_kernel_ms": round(decode_ms, 3), "decode_share": round(decode_ms / sum(kern.values()), 4),
        "outside_kernels_ms": round(prof_s * 1e3 - sum(kern.values()), 3),
        "fq_mul_per_proof_decode": muls_dec, "fq_mul_per_proof_verify": muls_ver,
        "count_ratio": round(muls_ver / (muls_ver + muls_dec), 3), "gpu": name, "power_limit": power,
        "invalid_checked": int((~want_ok).sum()),
    }))
    be.pvk_free(sim.pvk)
    be.close()


if __name__ == "__main__":
    main()
