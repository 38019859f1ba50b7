"""Per-kernel SASS instruction-class counts of libfluid_b200.so (cuobjdump -sass; no GPU needed).
usage: python tools/sass_counts.py [out.md]
Static counts of the whole kernel body (all paths), not executed counts: they prove which hardware
features a kernel is built from (LDGSTS, UTMALDG / mbarrier, shuffles, MUFU) and how big it is."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "webgl_fluid_simulation_b200", "libfluid_b200.so")
CLASSES = ["FADD", "FMUL", "FFMA", "MUFU", "SHFL", "LDG", "STG", "LDS", "STS", "LDGSTS", "UTMALDG",
           "UBLKCP", "SYNCS", "MOV", "BRA", "CALL", "HFMA2", "F2F", "F2FP", "DFMA"]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
    kernels, cur = collections.OrderedDict(), None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1); kernels[cur] = collections.Counter(); continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_]+)", line)
        if m and cur:
            kernels[cur][m.group(1)] += 1; kernels[cur]["_total"] += 1
    arch = subprocess.run(["cuobjdump", "-lelf", SO], capture_output=True, text=True).stdout
    demangle = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
    out = ["# SASS instruction-class counts per kernel of libfluid_b200.so (static, whole kernel body)", "",
           "cubins in the library: " + ", ".join(sorted(set(re.findall(r"sm_\d+a?", arch)))) + " (sm_90a only)", "",
           "| kernel | total | " + " | ".join(CLASSES) + " |", "|---|---|" + "---|" * len(CLASSES)]
    show = [k for k in kernels if re.search(r"tb_kernelILi10|cvd_stream|gradient_stream|advect_\w+4|splats_kernel|display|jacobi_sweep|jacobi8|halo_push|tiny_scan|curl_vorticity_div", k)]
    for k in show:
        c = kernels[k]
        name = re.sub(r"\(.*", "", demangle(k)).replace("fk::", "")
        out.append(f"| `{name}` | {c['_total']} | " + " | ".join(str(c[x]) if c[x] else "" for x in CLASSES) + " |")
    tot = collections.Counter()
    for c in kernels.values():
        tot.update(c)
    out += ["", f"whole library: {len(kernels)} kernels, {tot['_total']} instructions; " +
            ", ".join(f"{x} {tot[x]}" for x in ("SHFL", "LDGSTS", "UTMALDG", "UBLKCP", "SYNCS", "MUFU") if tot[x]) +
            f"; HGMMA {tot['HGMMA']} (no tensor-core instruction expected: there is no contraction on this path)"]
    text = "\n".join(out) + "\n"
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(text)
    else:
        print(text)


if __name__ == "__main__":
    main()
