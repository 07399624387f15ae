"""SASS opcode histogram of every kernel in the product library (no GPU needed):
    python tools/sass_histogram.py [path/to/libgh_raster.so] > <tag>_sass_opcodes.txt
Counts are STATIC instruction counts per kernel (cuobjdump -sass); the columns are the mnemonics that identify the
Hopper paths: LDGSTS (cp.async), UBLKCP + SYNCS (TMA bulk copy + mbarrier), REDG / RED (vector reductions to global
memory), MATCH, UCGABAR_ARV / _WAIT (cluster barrier), LDGMC (multimem.ld_reduce, NVLS)."""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "gaussianhaircut_b200", "lib", "libgh_raster.so")
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
names = subprocess.run(["cu++filt"], input="\n".join(re.findall(r"Function : (\S+)", sass)), capture_output=True, text=True).stdout.splitlines()
COLS = ["FFMA", "MUFU", "LDGSTS", "UBLKCP", "SYNCS", "REDG", "RED", "ATOMG", "ATOMS", "MATCH", "SHFL",
        "LDS", "STS", "LDG", "STG", "BAR", "UCGABAR*", "LDGMC", "DFMA", "FSEL"]
kernels, cur = [], None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = collections.Counter(); kernels.append(cur); continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
    if m and cur is not None:
        cur[m.group(1)] += 1; cur["_total"] += 1
print(f"# {os.path.basename(lib)}: static SASS instruction counts per kernel (cuobjdump -sass, sm_90a)")
print(f"{'kernel':46s} {'total':>6s} " + " ".join(f"{c:>7s}" for c in COLS))
for name, c in zip(names, kernels):
    short = re.sub(r"^.*?(gh_\w+).*$", r"\1", name)
    tmpl = re.search(r"<([^<>]*)>\(", name)
    if tmpl:
        short += "<" + tmpl.group(1).replace("(anonymous namespace)::", "") + ">"
    cnt = lambda k: sum(v for m, v in c.items() if m.startswith(k[:-1])) if k.endswith("*") else c.get(k, 0)  # noqa: E731
    print(f"{short[:46]:46s} {c['_total']:6d} " + " ".join(f"{cnt(k):7d}" for k in COLS))
