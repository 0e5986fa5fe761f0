"""Contexts on two devices in one process.  A kernel's dynamic shared-memory limit is a property of the device it is
raised on, so every device must raise it before its own first launch above the default 48 KiB, whichever device ran
the kernel first.  On each of devices 0 and 1 this runs plans on k_runs_tma (sorted row groups), k_tile_agg
(unsorted row groups; its ring of 6144-row stages of 8-byte columns alone is well above 48 KiB) and k_scan with
1024-row vectors (FROSTGPU_VL=1024: three ring slots of 8 KiB per staged column for each of its four warps), asserts
from the statistics which kernel took the row groups, and compares the results with the oracle and the reference.
Skipped with fewer than two visible GPUs."""
import os

import pytest
import torch

from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.store import ColumnStore
from tests import numeric_edges as ne
from tests.test_gpu_numeric_edges import N_RG, gpu_agg, oracle_agg, stats_of
from tests.test_gpu_parity import Pair

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")]

FILT = ne.leaf(ne.T, lp.OpGtEq, ne.RG // 2)  # a range leaf k_runs_tma takes
GENERAL = {"FROSTGPU_NO_RUNS": "1", "FROSTGPU_NO_TILE": "1", "FROSTGPU_VL": "1024"}


def test_large_shared_memory_launches_on_two_devices(built_lib):
    n_rows = 2 * ne.RG * len(ne.INT_CHUNKS)
    parts = [ne.int_part(ne.INT_CHUNKS, 21, sort=True), ne.int_part(ne.INT_CHUNKS, 22, sort=False, t0=n_rows // 2, part=1)]
    exp = ne.reference([ne.physical(c) for c in parts], FILT, ne.KEYS, ne.AGG_INT)
    for device in (0, 1):
        store = ColumnStore(device)
        p = Pair(store, f"launch_devices_{device}", dp.SampleDefinitionWithFloat())
        try:
            for cols, sort in zip(parts, (True, False)):
                buf = ne.write(cols, sort=sort, stats=False)  # nothing pruned: every row group is routed
                p.gt.InsertParquet(buf)
                p.ot.InsertParquet(buf)
            what = f"device {device}"
            ne.assert_same_result(oracle_agg(p, FILT, ne.KEYS, ne.AGG_INT), exp, ne.AGG_INT, what + " oracle")
            st = stats_of(store, p.name, FILT, ne.KEYS, ne.AGG_INT)
            assert (st["row_groups"], st["row_groups_runs"], st["row_groups_tiles"]) == (2 * N_RG, N_RG, N_RG), what
            ne.assert_same_result(gpu_agg(p, FILT, ne.KEYS, ne.AGG_INT), exp, ne.AGG_INT, what + " k_runs_tma + k_tile_agg")
            os.environ.update(GENERAL)
            try:
                st = stats_of(store, p.name, FILT, ne.KEYS, ne.AGG_INT)
                assert (st["row_groups"], st["row_groups_runs"], st["row_groups_tiles"]) == (2 * N_RG, 0, 0), what
                ne.assert_same_result(gpu_agg(p, FILT, ne.KEYS, ne.AGG_INT), exp, ne.AGG_INT, what + " k_scan")
            finally:
                for k in GENERAL:
                    os.environ.pop(k)
        finally:
            p.close()
            store.Close()
