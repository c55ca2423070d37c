"""SASS evidence per kernel of libbk200.so (cuobjdump -sass): instruction count and the mnemonics that prove the Hopper-native
paths (UBLKCP = cp.async.bulk / TMA bulk copy, SYNCS = mbarrier, FENCE.VIEW.ASYNC = fence.proxy.async, DFMA/DADD/DMUL = fp64 pipe,
LDS/STS = shared memory, LDG/STG = global, ACQBULK / griddepcontrol = PDL).   python tools/sass_summary.py   (prints the table)"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import sass_reader  # noqa: E402
so = sass_reader.library()
dem = lambda s: subprocess.run(["c++filt", s], capture_output=True, text=True).stdout.strip()
cnt = collections.OrderedDict()
for k, ops in sass_reader.opcodes(sass_reader.cuobjdump("-sass")).items():
    c = cnt[k] = collections.Counter(op.split(".")[0] for op in ops)
    c["FENCE.VIEW.ASYNC"] = sum(op.startswith("FENCE.VIEW.ASYNC") for op in ops)
    c["PDL"] = sum("ACQBULK" in op or "PREEXIT" in op or op.startswith("ACQ") for op in ops)
KEYS = ["UBLKCP", "UBLKPF", "SYNCS", "FENCE.VIEW.ASYNC", "DFMA", "DADD", "DMUL", "MUFU", "LDS", "STS", "LDG", "STG", "BAR", "LDL", "STL"]
print(f"# {os.path.relpath(so, ROOT)}: SASS mnemonic counts per kernel (sm_90a), from `cuobjdump -sass`")
print(f"{'instr':>7} " + " ".join(f"{k[:9]:>9}" for k in KEYS) + "  kernel")
tot = collections.Counter()
for k, c in sorted(cnt.items(), key=lambda kv: -sum(kv[1].values())):
    n = sum(v for kk, v in c.items() if kk not in ("FENCE.VIEW.ASYNC", "PDL"))
    name = re.sub(r"\(.*", "", dem(k))
    name = re.sub(r"^void ", "", name)
    print(f"{n:7d} " + " ".join(f"{c.get(kk, 0):9d}" for kk in KEYS) + f"  {name[:100]}")
    tot.update(c)
print("# totals: " + ", ".join(f"{k} {tot.get(k, 0)}" for k in KEYS) + f"; kernels {len(cnt)}")
