"""SASS evidence: per hot kernel of dedalus_b200/libdedalus_b200.so the counts of the instructions the design
claims rest on (UBLKCP = cp.async.bulk, SYNCS = mbarrier, LDGSTS = cp.async, DMMA = FP64 tensor core, DFMA/DADD/DMUL, LDS/STS,
BAR, SHFL, CCTL prefetch, STL/LDL local memory: spills and stack-resident locals).  usage: python scripts/sass_digest.py  (prints the digest as markdown)"""
import subprocess, re, collections, pathlib, sys
so = pathlib.Path(__file__).resolve().parents[1] / "dedalus_b200" / "libdedalus_b200.so"
out = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True).stdout
WANT = ["UBLKCP", "SYNCS", "LDGSTS", "DMMA", "DFMA", "DADD", "DMUL", "LDS", "STS", "LDG", "LD.E", "STG", "ST.E", "BAR", "SHFL", "CCTL", "FSEL", "BRA", "STL", "LDL"]
KERNELS = ["k_batches_solve_ws", "k_batches_solve_flat", "k_batches_solve_deep", "k_batches_matvec", "k_batches_move", "k_batches_factor",
           "k_batches_residual", "k_rbwd_regs", "k_rfwd_regs", "k_rfft_x_products", "k_chbwd_regs", "k_chfwd_regs", "k_pointwise_pairs", "k_mmt_dmma",
           "k_ragged_matvec", "k_band_scan2", "k_tr_chunks", "k_cfl_max"]
cur, counts, total = None, collections.OrderedDict(), {}
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1); counts[cur] = collections.Counter(); total[cur] = 0
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        op = m.group(1); total[cur] += 1
        for w in WANT:
            if op == w or op.startswith(w + ".") or (w in ("LD.E", "ST.E") and op.startswith(w)):
                counts[cur][w] += 1
print("# SASS digest of `dedalus_b200/libdedalus_b200.so` (sm_90a, `cuobjdump -sass`)\n")
print("Static instruction counts per kernel instance (not execution counts).  UBLKCP = `cp.async.bulk` (TMA engine, 1-D bulk copies of the solve's factor ring); SYNCS = mbarrier arrive / try_wait; LDGSTS = `cp.async`; DMMA = FP64 tensor-core MMA; CCTL = prefetch; STL / LDL = local-memory stores / loads.\n")
print("| kernel | instrs | " + " | ".join(WANT) + " |\n|---|---|" + "---|" * len(WANT))
import subprocess as sp
for fn, c in counts.items():
    if not any(k in fn for k in KERNELS):
        continue
    dem = sp.run(["c++filt", fn], capture_output=True, text=True).stdout.strip()
    dem = re.sub(r"\(.*$", "", dem.replace("(anonymous namespace)::", "")).replace("void ", "")
    if total[fn] < 40:
        continue
    print(f"| `{dem[:60]}` | {total[fn]} | " + " | ".join(str(c.get(w, 0)) for w in WANT) + " |")
