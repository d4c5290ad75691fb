"""Static resource table of every kernel (``nvcc -Xptxas -v``, cross-compiled for sm_90a; no GPU needed):
registers, static shared memory, spills, and the occupancy the register / launch-bound pair allows.

    python scripts/ptxas_resources.py        # -> profiles/ptxas_resources.md
"""
import os, re, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "federated-lifelong-person-reid_b200"))
import _build as B  # noqa: E402


def demangle(names):
    r = subprocess.run(["cu++filt", "-p"], input="\n".join(names), capture_output=True, text=True)
    out = r.stdout.strip().splitlines() if r.returncode == 0 else names
    return [x.replace("flpr::", "").replace("void ", "") for x in out]


def main():
    rows = []
    for src in B.CUDA_SOURCES:
        with tempfile.TemporaryDirectory() as tmp:
            cmd = [B._nvcc(), *B.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, src), "-o",
                   os.path.join(tmp, "x.o")]
            r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        cur = None
        for line in r.stderr.splitlines():
            m = re.search(r"Compiling entry function '([^']+)' for 'sm_90a'", line)
            if m:
                cur = {"src": src, "name": m.group(1), "spill_st": 0, "spill_ld": 0, "stack": 0}
                rows.append(cur)
                continue
            if cur is None:
                continue
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m:
                cur["stack"], cur["spill_st"], cur["spill_ld"] = map(int, m.groups())
            m = re.search(r"Used (\d+) registers(?:, used (\d+) barriers)?(?:, (\d+) bytes smem)?", line)
            if m:
                cur["regs"] = int(m.group(1))
                cur["bars"] = int(m.group(2) or 0)
                sm = re.search(r"(\d+) bytes smem", line)
                cur["smem"] = int(sm.group(1)) if sm else 0
    names = demangle([r["name"] for r in rows])
    out = ["# Kernel resources (`nvcc -Xptxas -v`, sm_90a)", "",
           "Static view of every `__global__` entry of `csrc/*.cu` (dynamic shared memory - the TMA stage rings of the",
           "wgmma kernels - is requested at launch and not part of this table). `spill` is stores/loads in bytes;",
           "the notes under the table say which instantiations run on the hot path.", "",
           "| source | kernel | regs | static smem (B) | barriers | stack (B) | spill st/ld (B) |", "|---|---|---|---|---|---|---|"]
    spills = 0
    for r, n in zip(rows, names):
        n = n if len(n) < 110 else n[:107] + "..."
        out.append(f"| {r['src']} | `{n}` | {r.get('regs', '?')} | {r.get('smem', 0)} | {r.get('bars', 0)} | {r['stack']} | "
                   f"{r['spill_st']}/{r['spill_ld']} |")
        spills += (r["spill_st"] + r["spill_ld"]) > 0
    out += ["", f"{len(rows)} entry points, {spills} with register spills.", "",
            "Notes", "",
            "* template arguments: `<BN, A operand mode, B operand mode, epilogue>`; operand modes 0 = K-major, 1 = MN-major,",
            "  2 = implicit-GEMM convolution (TMA im2col walk), 3 = tap-flipped convolution (dgrad)."]
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    path = os.path.join(ROOT, "profiles", "ptxas_resources.md")
    with open(path, "w") as f:
        f.write("\n".join(out) + "\n")
    print(path, len(rows), "kernels,", spills, "with spills")


if __name__ == "__main__":
    main()
