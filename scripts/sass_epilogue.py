"""Global-memory order of every gemm_wgmma_kernel instantiation in a built library (no GPU needed):
   python scripts/sass_epilogue.py [LIB_OR_OBJECT ...]     (default: the in-tree libomnitok_b200.so)

For each instantiation <TF32, NACC, EPI, H1> it lists the global loads (L, LDG) and stores (S, STG) in program order,
run-length encoded: "L4 S" is four loads then one store, and "(L2 S)x31" that pair of runs 31 times over.  `switches`
counts the load runs that follow a store.  An epilogue whose loads interleave with its stores pays one round trip to
L2 per switch, because the compiler may not move a load of a buffer that can alias the output above a store to it; an
epilogue that issues its loads in a batch shows a few switches per 64-row half."""
import argparse
import os
import re
import shutil
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KERNEL = re.compile(r"gemm_wgmma_kernelILb(\d)ELi(\d)ELi(\d)ELb(\d)E")
EPI_NAMES = {0: "plain", 1: "GEGLU", 2: "QKV", 3: "QKV planes"}


def cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        exe = "/usr/local/cuda/bin/cuobjdump"
    if exe is None:
        sys.exit("cuobjdump not found: put the CUDA toolkit's bin directory on PATH")
    return exe


def functions(path):
    """{mangled name: [SASS lines]} of every function in the file."""
    out = subprocess.run([cuobjdump(), "-sass", path], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
        elif cur is not None:
            cur.append(line)
    return funcs


def runs(lines):
    """[(kind, count)] of the global loads and stores in program order, consecutive ones of a kind merged."""
    seq = []
    for line in lines:
        m = re.search(r"\*/\s+(?:@!?U?P\w+\s+)?(LDG|STG)\.", line)
        if m is None:
            continue
        k = "L" if m.group(1) == "LDG" else "S"
        if seq and seq[-1][0] == k:
            seq[-1][1] += 1
        else:
            seq.append([k, 1])
    return [(k, n) for k, n in seq]


def compress(seq):
    """Runs as text, with a repeated (load run, store run) pair written once with its count."""
    tok = [f"{k}{n if n > 1 else ''}" for k, n in seq]
    pairs, i = [], 0
    while i < len(tok):
        if tok[i].startswith("L") and i + 1 < len(tok) and tok[i + 1].startswith("S"):
            pairs.append(f"{tok[i]} {tok[i + 1]}")
            i += 2
        else:
            pairs.append(tok[i])
            i += 1
    out, i = [], 0
    while i < len(pairs):
        j = i
        while j + 1 < len(pairs) and pairs[j + 1] == pairs[i]:
            j += 1
        n = j - i + 1
        out.append(f"({pairs[i]})x{n}" if n > 1 else pairs[i])
        i = j + 1
    return " ".join(out)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("paths", nargs="*", help="shared libraries or object files (default: the in-tree library)")
    args = ap.parse_args()
    paths = args.paths
    if not paths:
        from omnitokenizer_b200 import _cabi
        paths = [_cabi.lib_path()]
    for path in paths:
        print(f"{path}:")
        rows = []
        for name, lines in functions(path).items():
            m = KERNEL.search(name)
            if m is None:
                continue
            tf32, nacc, epi, h1 = (int(x) for x in m.groups())
            seq = runs(lines)
            loads = sum(n for k, n in seq if k == "L")
            stores = sum(n for k, n in seq if k == "S")
            switches = sum(1 for i in range(1, len(seq)) if seq[i][0] == "L" and seq[i - 1][0] == "S")
            tag = f"<{'true' if tf32 else 'false'}, {nacc}, {epi}{', true' if h1 else ''}>"
            rows.append((tf32, epi, nacc, h1, tag, EPI_NAMES.get(epi, str(epi)), loads, stores, switches, compress(seq)))
        for *_, tag, epi, loads, stores, switches, text in sorted(rows):
            print(f"  {tag:22s} {epi:10s} LDG {loads:4d}  STG {stores:4d}  switches {switches:3d}  {text}")


if __name__ == "__main__":
    main()
