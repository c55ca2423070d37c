"""The shipped library is sm_90a code and its hot kernels use the Hopper paths DESIGN.md claims: TMA bulk copies (SASS `UBLKCP`)
completing on mbarriers (`SYNCS`) in the fused JVP+Arnoldi ring kernels, fp64 FMAs, no local-memory spills there.  Read from the
built .so with cuobjdump (no GPU needed); tools/sass_summary.py prints the same counts."""
import re

import pytest

from tests import sass_reader as SR


@pytest.fixture(scope="module")
def sass():
    return SR.cuobjdump("--list-elf"), SR.mnemonics()


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
    ring = {k: u for k, u in SR.resources().items() if re.search(r"k2_(fused|update|dots)", k)}
    for k, u in ring.items():
        assert u.reg <= 56 and u.stack == 0, (k, u)
    assert len(ring) >= 32    # k2_fused<1..8, false / true>, k2_update<1..8>, k2_dots<1..8>
