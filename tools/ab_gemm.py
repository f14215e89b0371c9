"""A/B of two builds of libovg.so on one GPU: GEMM micro-benchmarks, bench.py cfg2 and cfg5, and byte-equal outputs.

    python tools/ab_gemm.py --build-parent REV       # on a build machine: libovg.so of commit REV -> build_ab/parent/
    python tools/ab_gemm.py [--rounds 3] [--out build_ab/ab_gemm]

Both builds run under the same Python tree (the C ABI is shared); the library is picked with OVG_LIB_PATH.  Every round runs, for
each build in turn (the order alternates between rounds so that a drift of the card's clocks does not favour one build):
tools/kbench.py's hot-path GEMMs (KB=gemm), then bench.py --config cfg2, then --config cfg5.  The first round also dumps the
outputs of cfg2 and cfg5 (bench.py --dump-outputs), and cfg3 is dumped once per build; every .npy must be byte-equal between the
builds.  Everything is written under --out; the summary is summary.json there and a table on stdout."""
from __future__ import annotations

import argparse
import filecmp
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "omnivggt-official_b200")
BUILDS = {"parent": os.path.join(ROOT, "build_ab", "parent", "libovg.so"), "new": os.path.join(PKG, "libovg.so")}


def build_parent(rev: str) -> str:
    """Compile libovg.so from the sources of commit `rev` with this tree's nvcc flags into build_ab/parent/."""
    sys.path.insert(0, PKG)
    import build as b
    out = BUILDS["parent"]
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        archive = subprocess.run(["git", "-C", ROOT, "archive", rev], check=True, capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", tmp], input=archive, check=True)
        src = os.path.join(tmp, "omnivggt-official_b200", "csrc", "ovg.cu")
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        r = subprocess.run([nvcc, *b.NVCC_FLAGS, "-o", out, src], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise SystemExit("nvcc failed building the parent libovg.so")
    with open(os.path.join(os.path.dirname(out), "REV"), "w") as f:
        f.write(subprocess.run(["git", "-C", ROOT, "rev-parse", rev], check=True, capture_output=True, text=True).stdout)
    return out


def run(cmd, env, log):
    """Run `cmd` from the repository root; its output goes to `log`.  Returns the last JSON line it printed (or None)."""
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise SystemExit(f"{' '.join(cmd)} failed ({r.returncode}); see {log}")
    for line in reversed(r.stdout.splitlines()):
        if line.startswith("{"):
            return json.loads(line)
    return None


def same_files(a: str, b: str):
    """(names that differ or exist on one side only, number of files compared)."""
    na, nb = set(os.listdir(a)), set(os.listdir(b))
    bad = sorted(na ^ nb)
    for n in sorted(na & nb):
        if not filecmp.cmp(os.path.join(a, n), os.path.join(b, n), shallow=False):
            bad.append(n)
    return bad, len(na & nb)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-parent", metavar="REV", help="build the parent libovg.so from commit REV and exit")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join("build_ab", "ab_gemm"))
    ap.add_argument("--cfg2-steps", type=int, default=10)
    ap.add_argument("--cfg5-steps", type=int, default=5)
    args = ap.parse_args()
    if args.build_parent:
        print(build_parent(args.build_parent))
        return
    for name, lib in BUILDS.items():
        if not os.path.exists(lib):
            raise SystemExit(f"missing {name} build {lib}")
    out = os.path.join(ROOT, args.out)
    shutil.rmtree(out, ignore_errors=True)
    os.makedirs(out)
    py = sys.executable
    bench_flags = ["--gpus", "1", "--no-cpu-baseline", "--no-gpu-torch-baseline"]
    kb = {b: [] for b in BUILDS}
    ms = {b: {"cfg2": [], "cfg5": []} for b in BUILDS}
    clocks = {b: {"cfg2": [], "cfg5": []} for b in BUILDS}
    for r in range(args.rounds):
        order = list(BUILDS) if r % 2 == 0 else list(reversed(BUILDS))
        for b in order:
            env = dict(os.environ, OVG_LIB_PATH=BUILDS[b], KB="gemm", KB_OUT=os.path.join(out, f"kbench_{b}_r{r}.json"))
            run([py, "tools/kbench.py"], env, os.path.join(out, f"kbench_{b}_r{r}.log"))
            kb[b].append(json.load(open(env["KB_OUT"])))
            for cfg, steps in (("cfg2", args.cfg2_steps), ("cfg5", args.cfg5_steps)):
                dump = ["--dump-outputs", os.path.join(out, f"dump_{cfg}_{b}")] if r == 0 else []
                line = run([py, "bench.py", *bench_flags, "--config", cfg, "--steps", str(steps), "--warmup", "3", *dump], env,
                           os.path.join(out, f"bench_{cfg}_{b}_r{r}.log"))
                ms[b][cfg].append(line["ms_per_step"])
                clocks[b][cfg].append(line.get("clocks"))
                print(f"round {r} {b:6s} {cfg}: {line['ms_per_step']:.2f} ms/step", flush=True)
    for b in BUILDS:
        env = dict(os.environ, OVG_LIB_PATH=BUILDS[b])
        run([py, "bench.py", *bench_flags, "--config", "cfg3", "--steps", "2", "--warmup", "3", "--dump-outputs",
             os.path.join(out, f"dump_cfg3_{b}")], env, os.path.join(out, f"bench_cfg3_{b}.log"))

    summary = {"card": kb["new"][0]["card"], "rounds": args.rounds, "outputs_byte_equal": {}, "bench": {}, "kbench": {}}
    ok = True
    for cfg in ("cfg2", "cfg3", "cfg5"):
        bad, n = same_files(os.path.join(out, f"dump_{cfg}_parent"), os.path.join(out, f"dump_{cfg}_new"))
        summary["outputs_byte_equal"][cfg] = {"files": n, "differ": bad}
        ok &= not bad and n > 0
        print(f"outputs {cfg}: {n} files, {'byte-equal' if not bad else 'DIFFER: ' + ', '.join(bad)}")
    for cfg in ("cfg2", "cfg5"):
        p, n = ms["parent"][cfg], ms["new"][cfg]
        d = dict(parent_ms=p, new_ms=n, parent_median=statistics.median(p), new_median=statistics.median(n),
                 parent_spread=max(p) - min(p), new_spread=max(n) - min(n),
                 change=statistics.median(n) / statistics.median(p) - 1.0, clocks={b: clocks[b][cfg] for b in BUILDS})
        summary["bench"][cfg] = d
        print(f"{cfg}: parent {d['parent_median']:.2f} ms (spread {d['parent_spread']:.2f}), new {d['new_median']:.2f} ms "
              f"(spread {d['new_spread']:.2f}), change {100 * d['change']:+.2f} %")
    print(f"{'GEMM':34s} {'parent ms':>10s} {'new ms':>10s} {'change':>8s} {'new TF/s':>9s} {'cuBLAS TF/s':>12s}")
    for k in kb["new"][0]:
        if not k.startswith("hot_"):
            continue
        p = statistics.median(x[k]["ms"] for x in kb["parent"])
        n = statistics.median(x[k]["ms"] for x in kb["new"])
        cub = statistics.median(x[k]["cublas_tflops"] for x in kb["new"] + kb["parent"])
        fl = 2.0 * kb["new"][0][k]["M"] * kb["new"][0][k]["N"] * kb["new"][0][k]["K"]
        summary["kbench"][k] = dict(parent_ms=p, new_ms=n, change=n / p - 1.0, parent_tflops=fl / p / 1e9, new_tflops=fl / n / 1e9,
                                    cublas_tflops=cub)
        print(f"{k:34s} {p:10.3f} {n:10.3f} {100 * (n / p - 1):+7.1f}% {fl / n / 1e9:9.1f} {cub:12.1f}")
    print("card:", json.dumps(summary["card"]))
    with open(os.path.join(out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    if not ok:
        raise SystemExit("outputs differ between the builds")


if __name__ == "__main__":
    main()
