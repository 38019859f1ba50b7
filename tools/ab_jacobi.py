"""Compare two builds of libfluid_b200.so on the pressure solve, alternated in one session.

usage: python tools/ab_jacobi.py OLD.so NEW.so [--runs 4] [--steps 2000] [--out DIR]

Every measurement is one `bench.py --quick` process with FLUID_B200_SO pointing at one of the two
libraries; old and new alternate run by run so that both see the same card, clocks and neighbours.
Printed: the card (name, power limit, max SM clock, from nvidia-smi), per run ms per solve with the
median SM clock and throttle reasons bench.py sampled, min / median / max per build, whether the
pressure fields of the two builds are byte-identical (--dump-outputs), and us per launch at single
depths (4 launches of depth K: --jacobi-block K --iters 4K), which shows which depths moved."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bench(so, extra, dump=None):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--quick"] + extra
    if dump:
        cmd += ["--dump-outputs", dump]
    env = dict(os.environ, FLUID_B200_SO=os.path.abspath(so))
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True).stdout
    return json.loads([l for l in out.splitlines() if l.startswith("{")][-1])


def sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def compare(name, libs, extra, runs, log):
    ms = {k: [] for k in libs}
    digest = {}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(runs):
            for k, so in libs.items():
                d = os.path.join(tmp, k) if r == 0 else None
                j = bench(so, extra, d)
                if d:
                    digest[k] = sha(os.path.join(d, "pressure.npy"))
                ms[k].append(j["ms_per_step"])
                c = j["clocks"]
                log(f"{name} run {r} {k}: {j['ms_per_step']:.4f} ms per solve, {j['roofline']['jacobi_launches_per_step']} launches, "
                    f"SM {c.get('sm_mhz')} MHz (max {c.get('sm_max_mhz')}), reasons {c.get('reasons')}")
    for k in libs:
        log(f"{name} {k}: min {min(ms[k]):.4f}  median {statistics.median(ms[k]):.4f}  max {max(ms[k]):.4f} ms per solve")
    old, new = statistics.median(ms["old"]), statistics.median(ms["new"])
    log(f"{name}: new / old medians = {new / old:.4f} ({100 * (1 - new / old):+.2f} % faster); new's slowest "
        f"{'<' if max(ms['new']) < min(ms['old']) else '>='} old's fastest; pressure fields "
        f"{'byte-identical' if digest['old'] == digest['new'] else 'DIFFER'}")
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old"); ap.add_argument("new")
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--depths-only", action="store_true", help="skip the two whole-solve comparisons")
    ap.add_argument("--out", default=None, help="directory for ab_jacobi.txt (default: print only)")
    a = ap.parse_args()
    libs = {"old": a.old, "new": a.new}
    lines = []

    def log(s):
        print(s, flush=True); lines.append(s)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    log("card: " + (q.stdout.strip() or "nvidia-smi gave nothing"))
    if not a.depths_only:
        compare("4096^2 x 50", libs, ["--steps", str(a.steps), "--warmup", "20"], a.runs, log)
        compare("8192^2 x 40", libs, ["--grid", "8192", "--iters", "40", "--steps", str(max(a.steps // 5, 1)), "--warmup", "10"],
                max(a.runs // 2, 1), log)
    for K in (9, 10, 12, 13):
        us = {k: [] for k in libs}
        for r in range(max(a.runs - 1, 1)):
            for k, so in libs.items():
                j = bench(so, ["--jacobi-block", str(K), "--iters", str(4 * K), "--steps", str(max(a.steps // 2, 1)), "--warmup", "20"])
                n = j["roofline"]["jacobi_launches_per_step"]
                us[k].append(1000 * j["ms_per_step"] / n)
                log(f"depth {K} run {r} {k}: {us[k][-1]:.1f} us per launch ({n} launches of {4 * K} sweeps), "
                    f"SM {j['clocks'].get('sm_mhz')} MHz, reasons {j['clocks'].get('reasons')}")
        log(f"depth {K}: old {min(us['old']):.1f}-{max(us['old']):.1f}, new {min(us['new']):.1f}-{max(us['new']):.1f} us per launch")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "ab_jacobi.txt"), "a").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
