"""CPU checks behind tests/test_gpu_cta.py: the numpy references of the block-wide primitives against brute force on
small exhaustive inputs, the key generators against what they promise, and the test harness built for sm_90a and kept
out of the product library."""
import itertools
import os
import subprocess

import numpy as np
import pytest

import cta_ref as R

HARNESS_SYMBOLS = ['cta_h_block_sizes', 'cta_h_scan', 'cta_h_warp_scan', 'cta_h_sort_u64', 'cta_h_sort_index',
                   'cta_h_radix_select', 'cta_h_smallest_sorted', 'cta_h_contract']


def _brute_select(keys, k, nbytes, bits):
    """By the definition: the least masked value v with at least k masked keys <= v, and how many of the first k keys in
    ascending order equal it."""
    shift = bits - 8 * nbytes
    masked = [(int(x) >> shift) << shift for x in keys]
    v = min(x for x in set(masked) if sum(y <= x for y in masked) >= k)
    return v, sorted(masked)[:k].count(v)


@pytest.mark.parametrize('bits', [32, 64])
def test_radix_select_reference_against_brute_force(bits):
    dtype = np.uint32 if bits == 32 else np.uint64
    top = 1 << (bits - 8)
    # values that differ in the top byte, in the lowest byte, in both, and the extremes
    alphabet = [0, 1, 0xFF, top, top + 1, 0xFF * top, (1 << bits) - 1, (1 << bits) - 2]
    nbytes_list = range(1, bits // 8 + 1)
    for n in range(1, 5):
        for keys in itertools.product(alphabet, repeat=n):
            arr = np.array(keys, dtype=dtype)
            for nbytes in nbytes_list:
                for k in range(1, n + 1):
                    key, rank = R.radix_select(arr, k, nbytes)
                    assert (int(key), rank) == _brute_select(keys, k, nbytes, bits), (keys, k, nbytes)


def test_radix_select_reference_rejects_k_outside_1_to_n():
    for k in (0, 4):
        with pytest.raises(AssertionError):
            R.radix_select(np.arange(3, dtype=np.uint32), k, 4)


def test_smallest_sorted_reference_against_brute_force():
    values = [0, 5, 9, 0xFFFFFFFFFFFFFFFE]
    for n in range(1, 5):
        for keys in itertools.permutations(values, n):
            for k in range(1, 7):
                got = R.smallest_sorted(np.array(keys, dtype=np.uint64), k)
                P = 1 << (k - 1).bit_length()
                want = sorted(keys)[:k] + [0xFFFFFFFFFFFFFFFF] * (P - min(k, n))
                assert [int(x) for x in got] == want, (keys, k)


def test_smallest_sorted_reference_asserts_the_preconditions():
    for keys, k in (([1, 1, 2], 2), ([1, 0xFFFFFFFFFFFFFFFF], 1), ([1, 2], 1025), ([1, 2], 0)):
        with pytest.raises(AssertionError):
            R.smallest_sorted(np.array(keys, dtype=np.uint64), k)


def test_scan_references():
    x = np.array([3, 0xFFFFFFFFFFFFFFFF, 2], dtype=np.uint64)
    assert R.inclusive_scan(x, 'sum').tolist() == [3, 2, 4]                    # mod 2^64
    assert R.exclusive_scan(x, 'sum', 0).tolist() == [0, 3, 2]
    y = np.array([-np.inf, -1.0, -np.inf, 2.0], dtype=np.float64)
    assert R.exclusive_scan(y, 'max', -np.inf).tolist() == [-np.inf, -np.inf, -1.0, -1.0]
    z = np.array([5, 3, 5], dtype=np.uint32)
    assert R.inclusive_scan(z, 'xor').tolist() == [5, 6, 3]


@pytest.mark.parametrize('dtype', [np.uint32, np.uint64])
def test_select_key_distributions(dtype):
    rng = np.random.default_rng(0)
    n, k = 5000, 2500
    for dist in R.DISTRIBUTIONS:
        keys = R.select_keys(dist, n, k, dtype, rng)
        assert keys.dtype == dtype and keys.shape == (n,), dist
    u = lambda d: np.unique(R.select_keys(d, n, k, dtype, rng))                # noqa: E731
    assert u('equal').size == 1
    assert np.unique(u('low_byte') >> dtype(8)).size == 1 and u('low_byte').size > 200
    assert np.unique(u('top_byte') & ~R.top_mask(dtype, 1)).size == 1 and u('top_byte').size > 200
    assert set(u('zero_ff').view(np.uint8).tolist()) == {0, 0xFF}
    dup = np.sort(R.select_keys('dup_at_k', n, k, dtype, rng))
    assert dup[k - 2] == dup[k - 1] == dup[k] and (dup == dup[k - 1]).sum() >= 64


def test_distinct_keys_cover_both_extremes():
    rng = np.random.default_rng(1)
    for n in (1, 2, 3, 1000):
        keys = R.distinct_keys(n, rng)
        assert keys.size == n and np.unique(keys).size == n and not (keys == R.ALL_ONES).any()
        if n >= 2:
            assert 0 in keys and np.uint64(0xFFFFFFFFFFFFFFFE) in keys


def _exports(path):
    out = subprocess.check_output(['nm', '-D', '--defined-only', path], text=True)
    return {line.split()[-1] for line in out.splitlines() if line.strip()}


@pytest.mark.skipif(not os.path.exists(os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')), reason='needs nvcc')
def test_harness_compiles_for_sm90a_and_exports_its_entry_points(tmp_path):
    from sipmask_b200 import build
    lib = build.build_cta_harness(out=str(tmp_path / 'libsmb_cta_harness.so'), force=True)
    assert set(HARNESS_SYMBOLS) <= _exports(lib)
    cuobjdump = os.path.join(os.path.dirname(build.NVCC), 'cuobjdump')
    elfs = subprocess.check_output([cuobjdump, '--list-elf', lib], text=True)
    assert 'sm_90a' in elfs and 'sm_' not in elfs.replace('sm_90a', '')


def test_product_library_exports_no_harness_symbol():
    from sipmask_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip('libsipmask_b200.so is not built')
    assert not {s for s in _exports(_lib.LIB_PATH) if s.startswith('cta_h_')}
