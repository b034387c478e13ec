"""numpy references of the block-wide primitives in sipmask_b200/csrc/cta.cuh, and the keys they are tested on
(tests/test_gpu_cta.py; the references themselves are checked against brute force in tests/test_cta_host.py).

Each reference asserts the primitive's preconditions, so a test can only ask the device what the header specifies."""
import numpy as np

# the block sizes tests/csrc/cta_harness.cu instantiates every kernel for (cta_h_block_sizes returns the same list)
BLOCK_SIZES = (32, 64, 96, 160, 256, 512, 992, 1024)
SELECT_CAP = 1024                       # the sel capacity of the harness's cta_smallest_sorted kernels
ALL_ONES = np.uint64(0xFFFFFFFFFFFFFFFF)
DISTRIBUTIONS = ('uniform', 'equal', 'low_byte', 'top_byte', 'zero_ff', 'dup_at_k')


def top_mask(dtype, nbytes):
    """The top `nbytes` bytes of a key of `dtype` (uint32 or uint64) set, the rest clear."""
    dtype = np.dtype(dtype)
    bits = 8 * dtype.itemsize
    assert dtype in (np.uint32, np.uint64) and 1 <= nbytes <= dtype.itemsize
    return dtype.type(((1 << bits) - 1) ^ ((1 << (bits - 8 * nbytes)) - 1))


def masked_sorted(keys, nbytes):
    keys = np.asarray(keys)
    return np.sort(keys & top_mask(keys.dtype, nbytes))


def select_from_sorted(masked, k):
    """cta_radix_select on keys whose masked, sorted values are `masked`: (the k-th smallest, its 1-based rank among the
    keys equal to it)."""
    assert 1 <= k <= masked.size, (k, masked.size)
    key = masked[k - 1]
    return key, k - int(np.searchsorted(masked, key, 'left'))


def radix_select(keys, k, nbytes):
    return select_from_sorted(masked_sorted(keys, nbytes), k)


def pow2_ceil(k):
    p = 1
    while p < k:
        p <<= 1
    return p


def smallest_sorted(keys, k, cap=SELECT_CAP):
    """cta_smallest_sorted's sel[0 .. P), P the next power of two of k: the min(k, n) smallest keys ascending, then
    ~0."""
    keys = np.asarray(keys, dtype=np.uint64)
    P = pow2_ceil(k)
    assert k >= 1 and keys.size >= 1 and P <= cap
    assert np.unique(keys).size == keys.size and not (keys == ALL_ONES).any(), 'distinct keys below ~0'
    out = np.full(P, ALL_ONES, dtype=np.uint64)
    s = np.sort(keys)[:k]
    out[:s.size] = s
    return out


def inclusive_scan(x, op):
    return {'sum': np.cumsum, 'max': np.maximum.accumulate, 'xor': np.bitwise_xor.accumulate}[op](x, dtype=x.dtype)


def exclusive_scan(x, op, identity):
    inc = inclusive_scan(x, op)
    return np.concatenate([np.array([identity], dtype=x.dtype), inc[:-1]])


def _uniform(rng, dtype, n):
    bits = 8 * np.dtype(dtype).itemsize
    return rng.integers(0, 1 << bits, n, dtype=np.uint64).astype(dtype)


def select_keys(dist, n, k, dtype, rng):
    """n keys of `dtype` drawn from one of DISTRIBUTIONS.  dup_at_k: uniform keys with the ones sorted around the k-th
    position replaced by the k-th, so a run of equal keys straddles it; the others do not depend on k."""
    dtype = np.dtype(dtype)
    bits = 8 * dtype.itemsize
    one = _uniform(rng, dtype, 1)[0]
    if dist == 'uniform':
        return _uniform(rng, dtype, n)
    if dist == 'equal':
        return np.full(n, one, dtype=dtype)
    if dist == 'low_byte':               # differ only in the lowest byte
        return (one & dtype.type(~dtype.type(0xFF))) | rng.integers(0, 256, n).astype(dtype)
    if dist == 'top_byte':               # differ only in the top byte
        top = rng.integers(0, 256, n).astype(dtype) << dtype.type(bits - 8)
        return (one & ~top_mask(dtype, 1)) | top
    if dist == 'zero_ff':                # every byte 0x00 or 0xFF: histogram bins 0 and 255 only
        return (rng.integers(0, 2, (n, dtype.itemsize)).astype(np.uint8) * np.uint8(0xFF)).view(dtype).reshape(n)
    if dist == 'dup_at_k':
        keys = _uniform(rng, dtype, n)
        order = np.argsort(keys, kind='stable')
        lo, hi = max(0, k - 33), min(n, k + 32)
        keys[order[lo:hi]] = keys[order[k - 1]]
        return keys
    raise ValueError(dist)


def distinct_keys(n, rng):
    """n distinct uint64 keys below ~0, in random order, including 0 and ~0 - 1 when n >= 2."""
    fixed = np.array([0, 0xFFFFFFFFFFFFFFFE], dtype=np.uint64)[:min(n, 2)]
    rest = np.unique(rng.integers(1, 0xFFFFFFFFFFFFFFFE, n + 64, dtype=np.uint64))
    rng.shuffle(rest)
    keys = np.concatenate([fixed, rest[:n - fixed.size]])
    assert keys.size == n
    rng.shuffle(keys)
    return keys
