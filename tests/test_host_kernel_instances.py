"""The instance table of tests/kernel_instances.py against the built library: the template instances of k_runs_tma,
k_tile_agg, k_take_count, k_take_write and k_runs_prefix in its device code (cuobjdump -symbols, demangled by cu++filt)
are exactly the table's tuples, reachable and unreachable; the fused pass's (NL, NK, NA, tight) tuples match the
dispatch limits of kernels.cu.  Adding or removing an instance without giving it a shape fails here."""
import os
import re
import shutil
import subprocess

import pytest

from tests import kernel_instances as ki

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = {"k_runs_tma": 168, "k_tile_agg": 64, "k_take_count": 6, "k_take_write": 24, "k_runs_prefix": 2}


def _tool(name):
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    path = os.path.join(cuda, "bin", name)
    return path if os.path.exists(path) else shutil.which(name)


@pytest.fixture(scope="module")
def device_symbols(built_lib):
    """Demangled names of every function in the library's device code."""
    from frostdb_b200 import _lib
    dump, filt = _tool("cuobjdump"), _tool("cu++filt")
    if not dump or not filt:
        pytest.skip("cuobjdump / cu++filt not found")
    out = subprocess.run([dump, "-symbols", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    names = [ln.split()[-1] for ln in out.splitlines() if "STT_FUNC" in ln]
    return subprocess.run([filt], input="\n".join(names), check=True, capture_output=True, text=True).stdout.splitlines()


def _arg(a: str):
    v = re.sub(r"^\((int|bool)\)", "", a.strip())
    return bool(int(v)) if a.strip().startswith("(bool)") else int(v)


def template_args(symbols, kernel: str, prefix: str = r"void fgpu::(<unnamed>|\(anonymous namespace\))::"):
    """The template-argument tuples of every instance of `kernel` (clones and callees of it not counted)."""
    rx = re.compile("^" + prefix + re.escape(kernel) + r"<([^>]*)>\(")
    return [tuple(_arg(a) for a in m.groups()[-1].split(",")) for m in map(rx.match, symbols) if m]


@pytest.mark.parametrize("kernel", sorted(SYMBOLS))
def test_compiled_instances_are_the_table(device_symbols, kernel):
    got = template_args(device_symbols, kernel)
    assert len(got) == len(set(got)) == SYMBOLS[kernel], f"{kernel}: {len(got)} instances in the library"
    table = set(ki.all_instances(kernel))
    assert set(got) == table, f"{kernel}: only in the library {sorted(set(got) - table)}, only in the table {sorted(table - set(got))}"


@pytest.mark.parametrize("kernel", ki.KERNELS)
def test_every_tuple_has_a_shape_or_a_reason(kernel):
    """Reachable tuples have at least one shape, whose plan the restated chooser maps to that tuple; unreachable ones
    have a reason and no shape."""
    shapes = ki.shapes(kernel)
    covered = {s.instance for s in shapes}
    unreachable = ki.UNREACHABLE[kernel]
    for s in shapes:
        assert ki.expected_instance(kernel, s) == s.instance, s.name()
    assert not covered & set(unreachable), sorted(covered & set(unreachable))
    assert all(reason for reason in unreachable.values())
    assert covered | set(unreachable) == set(ki.all_instances(kernel)), sorted(set(ki.all_instances(kernel)) - covered - set(unreachable))


def test_fused_pass_tuples_match_the_dispatch_limits(device_symbols):
    """fast_pass / fast_pass_tight are device functions of k_scan chosen per row group by fast_dispatch: NL 0..kFastLeaves,
    NK 0..kFastKeys, NA 0..kFastAggs, each in both variants."""
    src = open(os.path.join(ROOT, "frostdb_b200", "csrc", "kernels.cu")).read()
    m = re.search(r"constexpr int kFastLeaves = (\d+), kFastKeys = (\d+), kFastAggs = (\d+);", src)
    assert m, "kFastLeaves / kFastKeys / kFastAggs not found in kernels.cu"
    assert tuple(map(int, m.groups())) == (ki.FAST_LEAVES, ki.FAST_KEYS, ki.FAST_AGGS)
    table = set(ki.all_instances("fast_pass"))
    assert len(table) == 72
    # the symbols, where the compiler kept the device functions as calls (they are __noinline__)
    clone = r"\[clone fgpu::k_scan\(const fgpu::QueryDesc \*\)\] unsigned int fgpu::"
    tight = {a + (True,) for a in template_args(device_symbols, "fast_pass_tight", clone)}
    loose = {a + (False,) for a in template_args(device_symbols, "fast_pass", clone)}
    if tight or loose:
        assert tight | loose == table, sorted((tight | loose) ^ table)
