"""The periodic transform modes (bk_fft_fast.cuh: k_contig MODE 2 / 3, k_strided MODE 3) are in the sm_90a library, stage their
tables with bulk copies completing on an mbarrier, and spill nothing to local memory in the instantiations the library launches
(values per thread E = 4 below n = 1024, E = 8 from 1024 on; bk_precond.cu::fast_loge).  Read with cuobjdump, no GPU needed."""
import re

import pytest

from tests import sass_reader as SR


@pytest.fixture(scope="module")
def sass():
    return SR.cuobjdump("--list-elf"), SR.mnemonics()


def _periodic(cnt):
    """(kernel, log2 n, log2 E, mode) -> counts of the periodic modes"""
    res = {}
    for k, c in cnt.items():
        m = re.search(r"(k_contig|k_strided)INS_3CfgILi(\d+)ELi(\d)EEELi(\d)EE", k)
        if not m:
            continue
        key = (m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4)))
        if (key[0] == "k_contig" and key[3] in (2, 3)) or (key[0] == "k_strided" and key[3] == 3):
            res[key] = c
    return res


def test_periodic_modes_exist_in_the_sm_90a_cubin(sass):
    elfs, cnt = sass
    assert all(".sm_90a." in n for n in re.findall(r"ELF file\s+\d+:\s+(\S+)", elfs))
    per = _periodic(cnt)
    for logn in range(6, 12):
        for loge in (2, 3, 4, 5):
            for key in (("k_contig", logn, loge, 2), ("k_contig", logn, loge, 3), ("k_strided", logn, loge, 3)):
                assert key in per, key


def test_periodic_modes_use_bulk_copies_and_mbarriers(sass):
    _, cnt = sass
    for key, c in _periodic(cnt).items():
        assert c["UBLKCP"] >= 2 and c["SYNCS"] >= 1 and c["DFMA"] >= 10, (key, dict(c))


def test_launched_periodic_instantiations_do_not_spill(sass):
    _, cnt = sass
    per = _periodic(cnt)
    for logn in range(6, 12):
        loge = 3 if logn >= 10 else 2
        for key in (("k_contig", logn, loge, 2), ("k_contig", logn, loge, 3), ("k_strided", logn, loge, 3)):
            c = per[key]
            assert c["LDL"] == 0 and c["STL"] == 0, (key, dict(c))
