"""A/B of the compositors against a parent build of the library, in one run on one GPU.

The parent arm loads another build of libr3dg_b200.so through R3DG_LIB_PATH (default variants/parent/, git-ignored;
build it from the parent commit with `python -m relightable3dgaussian_b200.build` in a checkout of that commit and copy
the .so there).  Runs, alternating the arms:
  * bench.py --gpus 1 --steps 200 --warmup 10 --no-cpu-baseline, `--runs` times per arm: `value` and every stage of
    `stage_ms`, with their medians per arm;
  * tools/bench_views.py at one view (its 1M/800x800/S=5 and 1.5M/1600x1200/S=16 shapes), bench_deterministic.py,
    bench_absgrad.py and bench_frozen_geometry.py, `--other-runs` times per arm;
  * bench.py --dump-outputs for each arm (and a second parent run, the parent's own run-to-run spread), compared:
    images and counts bitwise, per-Gaussian gradients by relative L2.
Prints every result line as it comes and the summary at the end (with `--out FILE`, also writes them to FILE as JSON
lines); the device name, power limit and maximum SM clock are read in the same run.

    python tools/bench_composite.py [--parent variants/parent/libr3dg_b200.so] [--runs 3] [--other-runs 1]
                                    [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_json(cmd, lib):
    env = dict(os.environ)
    if lib:
        env["R3DG_LIB_PATH"] = lib
    else:
        env.pop("R3DG_LIB_PATH", None)
    r = subprocess.run([sys.executable] + cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"{cmd} failed ({r.returncode}):\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    return json.loads(lines[-1])


def compare_dumps(a, b):
    import numpy as np
    out = {}
    for f in sorted(os.listdir(a)):
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        name = f[:-4]
        if name.startswith("grad_"):
            den = float(np.linalg.norm(x.astype(np.float64)))
            out[name] = float(np.linalg.norm(x.astype(np.float64) - y)) / den if den > 0 else float(np.abs(y).max())
        else:
            out[name] = "bitwise" if np.array_equal(x, y, equal_nan=True) else f"max|d| {float(np.nanmax(np.abs(x - y)))}"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=os.path.join(ROOT, "variants", "parent", "libr3dg_b200.so"))
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--other-runs", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the result lines and the summary here (JSON lines)")
    args = ap.parse_args()
    if not os.path.exists(args.parent):
        sys.exit(f"no parent build at {args.parent}")
    log = open(args.out, "w") if args.out else None

    def rec(d):
        print(json.dumps(d), flush=True)
        if log:
            log.write(json.dumps(d) + "\n")
            log.flush()

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    summary = {"device": smi}
    arms = {"parent": args.parent, "branch": None}
    headline = ["bench.py", "--gpus", "1", "--steps", "200", "--warmup", "10", "--no-cpu-baseline"]
    res = {a: [] for a in arms}
    for i in range(args.runs):
        for a in (("parent", "branch") if i % 2 == 0 else ("branch", "parent")):
            r = run_json(headline, arms[a])
            rec({"arm": a, "workload": "headline", "result": r})
            res[a].append({"value": r["value"], **{f"{k}_ms": v for k, v in r["stage_ms"].items()}})
    summary["headline"] = res
    for a in arms:
        summary[f"headline_{a}_median"] = {k: statistics.median(x[k] for x in res[a]) for k in res[a][0]}
    others = {"views": ["tools/bench_views.py", "--views", "1", "--rounds", "1"],
              "deterministic": ["tools/bench_deterministic.py"],
              "absgrad": ["tools/bench_absgrad.py"],
              "frozen_geometry": ["tools/bench_frozen_geometry.py"]}
    for name, cmd in others.items():
        for i in range(args.other_runs):
            for a in (("parent", "branch") if i % 2 == 0 else ("branch", "parent")):
                rec({"arm": a, "workload": name, "result": run_json(cmd, arms[a])})
    with tempfile.TemporaryDirectory() as tmp:
        dumps = {}
        for a in ("parent", "branch", "parent2"):
            dumps[a] = os.path.join(tmp, a)
            run_json(headline[:4] + ["20", "--warmup", "2", "--no-cpu-baseline", "--dump-outputs", dumps[a]],
                     arms["parent" if a == "parent2" else a])
        summary["outputs_branch_vs_parent"] = compare_dumps(dumps["parent"], dumps["branch"])
        summary["outputs_parent_vs_parent"] = compare_dumps(dumps["parent"], dumps["parent2"])
    rec({"summary": summary})
    print(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
