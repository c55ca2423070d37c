"""The shipped library is sm_90a code and its hot kernels use the Hopper paths DESIGN.md claims: TMA bulk copies (SASS `UBLKCP`)
completing on mbarriers (`SYNCS`) in the fused JVP+Arnoldi ring kernels, fp64 FMAs, no local-memory spills there.  Read from the
built .so with cuobjdump (no GPU needed); tools/sass_summary.py prints the same counts."""
import collections
import os
import re
import shutil
import subprocess

import pytest

import __graft_entry__ as g


@pytest.fixture(scope="module")
def sass():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    bk = g.load_package()
    if not os.path.exists(bk.lib.LIB_PATH):
        bk.build()
    elfs = subprocess.run(["cuobjdump", "--list-elf", bk.lib.LIB_PATH], capture_output=True, text=True).stdout
    out = subprocess.run(["cuobjdump", "-sass", bk.lib.LIB_PATH], capture_output=True, text=True).stdout
    cnt, cur = {}, None
    for l in out.splitlines():
        m = re.search(r"Function : (\S+)", l)
        if m:
            cur = m.group(1)
            cnt[cur] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_.]+)", l)
        if m and cur:
            cnt[cur][m.group(2).split(".")[0]] += 1
    return elfs, cnt


def test_every_cubin_is_sm_90a(sass):
    elfs, _ = sass
    names = re.findall(r"ELF file\s+\d+:\s+(\S+)", elfs)
    assert len(names) >= 6 and all(".sm_90a." in n for n in names), names


def test_ring_kernels_use_tma_bulk_copies_and_mbarriers(sass):
    _, cnt = sass
    ring = {k: c for k, c in cnt.items() if re.search(r"k2_(fused|update|dots|apply)", k)}
    assert len(ring) >= 20, sorted(ring)[:5]          # every tile height E = 1..8 of k2_fused<E, bordered>, k2_update<E>, k2_dots<E>, k2_apply<E, MODE>
    for k, c in ring.items():
        assert c["UBLKCP"] >= 1 and c["SYNCS"] >= 1, (k, dict(c))    # cp.async.bulk + mbarrier
        assert c["DFMA"] >= 1 and c["LDL"] == 0 and c["STL"] == 0, (k, dict(c))  # fp64 pipe, nothing spilled to local memory
    fused = [c for k, c in ring.items() if "k2_fused" in k]
    assert all(c["UBLKPF"] >= 1 for c in fused)                        # L2 prefetch of the u / a / b rows (cp.async.bulk.prefetch)
    # the ring kernels are the only Arnoldi kernels: no non-ring JVP+dots, dots or update kernel is built
    old = [k for k in cnt if re.search(r"(?<!\d)(16k_fused_jvp_dots|6k_dots|13k_update_norm)", k)]
    assert not old, old


def test_transform_kernels_stage_their_tables_by_bulk_copy(sass):
    _, cnt = sass
    tr = {k: c for k, c in cnt.items() if re.search(r"k_strided|k_contig", k)}
    assert len(tr) >= 30
    for k, c in tr.items():
        assert c["UBLKCP"] >= 2 and c["SYNCS"] >= 1 and c["DFMA"] >= 10, (k, dict(c))


def test_ring_kernels_fit_four_ctas_per_sm():
    """bk_krylov.cu plans BK2_BLOCKS_PER_SM = 4 CTAs of 288 threads per SM (grid sizing, shared-memory budget): that needs
    <= 65536 / (4 x 288) = 56 registers per thread and no stack frame; read from the built library (cuobjdump --dump-resource-usage)"""
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    bk = g.load_package()
    out = subprocess.run(["cuobjdump", "--dump-resource-usage", bk.lib.LIB_PATH], capture_output=True, text=True).stdout
    seen = 0
    fn = None
    for l in out.splitlines():
        m = re.search(r"Function (\S+):", l)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"REG:(\d+)\s+STACK:(\d+)", l)
        if m and fn and re.search(r"k2_(fused|update|dots)", fn):
            assert int(m.group(1)) <= 56 and int(m.group(2)) == 0, (fn, l.strip())
            seen += 1
            fn = None
    assert seen >= 32    # k2_fused<1..8, false / true>, k2_update<1..8>, k2_dots<1..8>
