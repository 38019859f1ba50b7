"""Compile and run tools/stage_probe.cu on cuda:0: staging-only launches against the depth-13 blocked kernel.

usage: python tools/stage_probe.py [--launches 1000] [--repeats 3] [--out DIR]

The probe is built into a temporary directory with the library's nvcc flags (sm_90a).  The card's name,
power limit and maximum SM clock are printed before the run, and the SM clock is sampled by nvidia-smi
every 200 ms while it runs (min / median / max printed after it)."""
import argparse
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--fmad=false", "-prec-div=true",
         "-prec-sqrt=true", "-ftz=false", "-Xptxas", "-v"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for stage_probe.txt (default: print only)")
    a = ap.parse_args()
    lines = []

    def log(s):
        print(s, flush=True); lines.append(s)

    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "stage_probe")
        b = subprocess.run([NVCC] + FLAGS + ["-o", exe, os.path.join(ROOT, "tools", "stage_probe.cu")],
                           capture_output=True, text=True)
        for l in b.stderr.splitlines():
            if "registers" in l or "spill" in l or "error" in l:
                log("ptxas: " + l.strip())
        if b.returncode:
            sys.exit(b.stderr)
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        log("card: " + (q.stdout.strip() or "nvidia-smi gave nothing"))
        smp = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms", "200"],
                               stdout=subprocess.PIPE, text=True)
        try:
            r = subprocess.run([exe, str(a.launches), str(a.repeats)], capture_output=True, text=True)
        finally:
            smp.terminate()
            clk = smp.communicate(timeout=10)[0]
        for l in r.stdout.splitlines():
            log(l)
        if r.stderr:
            log(r.stderr.strip())
        mhz = [int(x) for x in clk.split() if x.isdigit()]
        if mhz:
            log(f"SM clock during the run: min {min(mhz)}  median {statistics.median(mhz)}  max {max(mhz)} MHz ({len(mhz)} samples)")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "stage_probe.txt"), "a").write("\n".join(lines) + "\n")
    sys.exit(r.returncode)


if __name__ == "__main__":
    main()
