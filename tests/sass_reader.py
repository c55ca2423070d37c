"""The sm_90a code of the built libbk200.so as cuobjdump shows it, read without a GPU: the SASS mnemonics and the resource usage
(registers, stack, local memory) of every kernel.  The SASS tests read the library through this module; tools/sass_summary.py
prints its counts."""
import collections
import functools
import os
import re
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

Usage = collections.namedtuple("Usage", "reg stack local")


def library():
    """the path of libbk200.so, built first if it is missing"""
    import __graft_entry__ as g
    bk = g.load_package()
    if not os.path.exists(bk.lib.LIB_PATH):
        bk.build()
    return bk.lib.LIB_PATH


@functools.lru_cache(maxsize=None)
def cuobjdump(flag):
    """the output of `cuobjdump <flag>` on the library; skips the calling test where cuobjdump is not on PATH"""
    if shutil.which("cuobjdump") is None:
        import pytest
        pytest.skip("cuobjdump not on PATH")
    return subprocess.run(["cuobjdump", flag, library()], capture_output=True, text=True).stdout


def opcodes(sass):
    """kernel (mangled name) -> the opcodes of its instructions in `cuobjdump -sass` output, with their modifiers (LDG.E.64)"""
    ops, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            ops[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and cur:
            ops[cur].append(m.group(2))
    return ops


def mnemonics():
    """kernel -> counts of the mnemonics (opcodes without modifiers) of its SASS"""
    return {k: collections.Counter(o.split(".")[0] for o in ops) for k, ops in opcodes(cuobjdump("-sass")).items()}


def resources():
    """kernel -> Usage(reg, stack, local) from `cuobjdump --dump-resource-usage` (bytes for stack and local)"""
    res, fn = {}, None
    for line in cuobjdump("--dump-resource-usage").splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"REG:(\d+)\s+STACK:(\d+).*LOCAL:(\d+)", line)
        if m and fn:
            res[fn] = Usage(*map(int, m.groups()))
            fn = None
    return res
