"""The benchmarked Groth16 proof (bench.py's DummyCircuit shape and synthetic key) with a uniform witness instead of the
all-equal one, with the h-query table on and off.

bench.py's witness repeats one value, so the multiplicity-aware front end turns the a, b_g1, b_g2 and l MSMs into a few
heavy lists and only the h MSM pays the full Pippenger price.  Here every witness entry is a random scalar: z no longer
satisfies the constraints, but the witness map and the prover are defined for every assignment, and the proof is still
checked against its known discrete logs (bench.py's verify_proof).  All five MSMs then run the full pipeline, the G2 one
with the largest batched-affine round scratch of the proof; with the table resident those rounds may run in slices.

  python tools/uniform_prove_probe.py --log-n 24 --rounds 2 --steps 3 --warmup 1

Each (round, mode) is its own process (the table is built at key upload, so B2S_PK_PRECOMP=0 needs a fresh key), modes
alternated.  Prints the card's name and power limit, then one line per process and a summary of ms per proof and of the G2
kernels of the profiled pass."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED_UNIFORM = 0x0F0E0D0C


def child(argv):
    """bench.py's GPU arm with a uniform witness; the result line of bench.py goes to stdout."""
    sys.path.insert(0, ROOT)
    import bench
    from tests.util import random_fr_limbs

    plain = bench.dummy_instance

    def uniform_instance(log_n):
        inst = plain(log_n)
        rng = np.random.default_rng(SEED_UNIFORM)
        inst["z_inst"][8:16] = random_fr_limbs(rng, 1, bits=253)        # z[0] = 1 stays; Montgomery forms of values < r
        inst["z_wit"] = random_fr_limbs(rng, inst["n_wit"], bits=253)
        return inst

    bench.dummy_instance = uniform_instance
    # h of a non-satisfying z is still a defined function of z, but the comparison with the CPU oracle's witness map is not
    # what this probe is about and costs a minute at 2^24: the proof is checked against its known discrete logs only
    verify = bench.verify_proof
    bench.verify_proof = lambda *a, **k: verify(*a, **{**k, "check_h": False})
    sys.argv = ["bench.py", "--gpus", "1", "--no-cpu", "--no-extras"] + argv
    bench.main()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--save", metavar="DIR", help="also write each process's bench.py result line to DIR/<mode>_<round>.json")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args, rest = ap.parse_known_args()
    bench_args = ["--log-n", str(args.log_n), "--steps", str(args.steps), "--warmup", str(args.warmup)]
    if args.child:
        child(bench_args + rest)
        return
    print("card:", card(), flush=True)
    results = {"table": [], "no_table": []}
    for rnd in range(args.rounds):
        for mode in ("table", "no_table"):
            env = dict(os.environ)
            env.pop("B2S_PK_PRECOMP", None)
            if mode == "no_table":
                env["B2S_PK_PRECOMP"] = "0"
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"] + bench_args, env=env, cwd=ROOT, capture_output=True, text=True)
            line = p.stdout.strip().splitlines()[-1] if p.stdout.strip() else ""
            if p.returncode != 0 or not line.startswith("{"):
                sys.stderr.write(p.stderr[-4000:])
                raise SystemExit(f"{mode} round {rnd}: exit {p.returncode}")
            out = json.loads(line)
            if args.save:
                os.makedirs(args.save, exist_ok=True)
                with open(os.path.join(args.save, f"{mode}_{rnd}.json"), "w") as f:
                    f.write(line + "\n")
            kern = out["kernel_ms_per_step"]
            g2 = {k: v for k, v in kern.items() if k.endswith("_g2")}
            rec = {"round": rnd, "mode": mode, "ms_per_step": round(out["ms_per_step"], 2), "verified": out["verified"],
                   "kernel_ms_total": round(sum(kern.values()), 2),
                   "msm_ba_g2_ms": round(sum(v for k, v in g2.items() if k.startswith("msm_ba_")), 2),
                   "msm_accumulate_g2_ms": g2.get("msm_accumulate_g2"), "h_table_kernels": {k: kern[k] for k in kern if "bucket" in k or "window" in k}}
            print(json.dumps(rec), flush=True)
            assert out["verified"] and out["verified"]["proof_equals_known_discrete_logs"], "proof does not match its known discrete logs"
            results[mode].append(out["ms_per_step"])
    print("card:", card())
    print(json.dumps({m: {"ms_per_step": [round(v, 2) for v in vs], "median": round(float(np.median(vs)), 2)} for m, vs in results.items()}))


if __name__ == "__main__":
    main()
