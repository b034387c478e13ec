"""The block-wide primitives of sipmask_b200/csrc/cta.cuh on their own (through the test harness
tests/csrc/cta_harness.cu, libsmb_cta_harness.so), at every block size of the harness's table and every key width, bit
for bit against the numpy references of tests/cta_ref.py; then the consumer kernels where a primitive's carry crosses a
chunk: pair_select_kernel's tie budget, finalize_kernel's class-offset scan and the RLE kernels' offset scans.

Every comparison is exact.  Device calls stay inside each primitive's preconditions (the references assert them)."""
import ctypes

import numpy as np
import pytest
import torch

import cta_ref as R

pytestmark = pytest.mark.gpu

U64 = np.uint64


@pytest.fixture(scope='module')
def H():
    from sipmask_b200 import build
    L = ctypes.CDLL(build.CTA_HARNESS_LIB)
    sizes = (ctypes.c_int * 16)()
    n = L.cta_h_block_sizes(sizes, 16)
    assert tuple(sizes[:n]) == R.BLOCK_SIZES
    return L


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(rc):
    assert rc == 0, 'harness launch failed with cudaError %d' % rc


def _dev(a):
    """numpy -> CUDA tensor of the same bits (unsigned types travel as the signed type of their width)."""
    a = np.ascontiguousarray(a)
    view = {np.dtype(np.uint64): np.int64, np.dtype(np.uint32): np.int32}.get(a.dtype, a.dtype)
    return torch.from_numpy(a.view(view).copy()).cuda()


def _host(t, dtype):
    return t.cpu().numpy().view(dtype)


# ------------------------------------------------------------------------------------------------ scans

SCAN_OPS = {  # op code of cta_h_scan, dtype, reference op, identity
    'i32_sum': (0, np.int32, 'sum', 0),
    'u64_sum': (1, np.uint64, 'sum', 0),
    'f64_max': (2, np.float64, 'max', -np.inf),
    'u32_xor': (3, np.uint32, 'xor', 0),
}


def _scan_input(name, threads, blocks, rng):
    n = threads * blocks
    if name == 'i32_sum':
        return rng.integers(-(1 << 20), 1 << 20, n).astype(np.int32)
    if name == 'u64_sum':                       # wraps mod 2^64 within a few threads
        return rng.integers(0, 1 << 64, n, dtype=np.uint64)
    if name == 'u32_xor':
        return rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    x = rng.standard_normal(n)                   # the precision envelope's entries: -1 and -inf among the values
    x[rng.random(n) < 0.2] = -1.0
    x[rng.random(n) < 0.1] = -np.inf
    x[:threads] = -np.inf                        # one segment with nothing but -inf
    x[threads:threads + 40] = -1.0               # and one that starts with a run of -1
    return x


@pytest.mark.parametrize('name', list(SCAN_OPS))
@pytest.mark.parametrize('threads', R.BLOCK_SIZES)
def test_cta_scans(H, name, threads):
    op, dtype, ref_op, identity = SCAN_OPS[name]
    blocks = 5
    x = _scan_input(name, threads, blocks, np.random.default_rng(threads * 7 + op))
    assert x.dtype == dtype
    d_in = _dev(x)
    outs = [torch.empty_like(d_in) for _ in range(4)]
    _ok(H.cta_h_scan(op, threads, blocks, _p(d_in), *[_p(o) for o in outs], _st()))
    inc, exc, tot_inc, tot_exc = [_host(o, dtype).reshape(blocks, threads) for o in outs]
    for b, seg in enumerate(x.reshape(blocks, threads)):
        want = R.inclusive_scan(seg, ref_op)
        assert np.array_equal(inc[b], want), (b, np.nonzero(inc[b] != want)[0][:5])
        assert np.array_equal(exc[b], R.exclusive_scan(seg, ref_op, identity)), b
        assert (tot_inc[b] == want[-1]).all() and (tot_exc[b] == want[-1]).all(), b


@pytest.mark.parametrize('lanes', [1, 2, 3, 7, 8, 31, 32])
def test_warp_inclusive_scan(H, lanes):
    warps = 8
    x = np.random.default_rng(lanes).integers(-1000, 1000, warps * 32).astype(np.int32)
    d_in = _dev(x)
    out = torch.empty_like(d_in)
    _ok(H.cta_h_warp_scan(lanes, warps, _p(d_in), _p(out), _st()))
    got = _host(out, np.int32).reshape(warps, 32)[:, :lanes]        # lanes >= kLanes are unspecified
    assert np.array_equal(got, np.cumsum(x.reshape(warps, 32), axis=1, dtype=np.int32)[:, :lanes])


# ------------------------------------------------------------------------------------------------ bitonic sort

SORT_P = [1 << e for e in range(14)]                # 1 .. 8192; 8192 u64 keys are 64 KB of dynamic shared memory


def _sort_segments(P, rng):
    """Random keys with duplicates, random full-range keys, sorted, reversed and constant input."""
    dup = rng.integers(0, max(2, P // 4), P, dtype=np.uint64)
    full = rng.integers(0, 1 << 64, P, dtype=np.uint64)
    return np.stack([dup, full, np.sort(full), np.sort(full)[::-1], np.full(P, full[0])])


@pytest.mark.parametrize('P', SORT_P)
def test_cta_bitonic_sort_u64(H, P):
    segs = _sort_segments(P, np.random.default_rng(P))
    d_in = _dev(segs.reshape(-1))
    out = torch.empty_like(d_in)
    for threads in R.BLOCK_SIZES:                   # wider and narrower than the P / 2 comparators of a step
        out.fill_(0)
        _ok(H.cta_h_sort_u64(P, threads, segs.shape[0], _p(d_in), _p(out), _st()))
        got = _host(out, U64).reshape(segs.shape)
        for b in range(segs.shape[0]):
            assert np.array_equal(got[b], np.sort(segs[b])), (threads, b)


@pytest.mark.parametrize('P', SORT_P)
def test_cta_bitonic_sort_index_through_key_table(H, P):
    """match2_kernel's order: rows by descending key from a table, ties by row, the -1 padding after every row."""
    rng = np.random.default_rng(P + 1)
    n_valid = sorted({P, P - 1, P // 2 + 1, 1, 0})
    keys = rng.choice(np.float32([0.25, 0.5, 0.75, 1.0]), (len(n_valid), P))       # many ties
    d_key, d_nv = _dev(keys.reshape(-1)), _dev(np.int32(n_valid))
    out = torch.empty(len(n_valid) * P, dtype=torch.int32, device='cuda')
    for threads in R.BLOCK_SIZES:
        out.fill_(-7)
        _ok(H.cta_h_sort_index(P, threads, len(n_valid), _p(d_key), _p(d_nv), _p(out), _st()))
        got = _host(out, np.int32).reshape(len(n_valid), P)
        for b, nv in enumerate(n_valid):
            rows = np.arange(nv)
            want = np.concatenate([np.lexsort((rows, -keys[b, :nv])), np.full(P - nv, -1)])
            assert np.array_equal(got[b], want), (threads, nv)


# ------------------------------------------------------------------------------------------------ radix select

SELECT_WIDTHS = [(32, b) for b in range(1, 5)] + [(64, b) for b in range(1, 9)]


class _KeyPool:
    """Every key array a test's queries read, concatenated into one device buffer, with each array's masked sort."""

    def __init__(self, dtype, rng):
        self.dtype, self.rng, self.parts, self.index, self.size = dtype, rng, [], {}, 0
        self._sorted = {}

    def add(self, dist, n, k):
        tag = (dist, n, k if dist == 'dup_at_k' else 0)
        if tag not in self.index:
            keys = R.select_keys(dist, n, k, self.dtype, self.rng)
            self.index[tag] = (self.size, keys)
            self.parts.append(keys)
            self.size += n
        return tag

    def offset(self, tag):
        return self.index[tag][0]

    def masked_sorted(self, tag, nbytes):
        if (tag, nbytes) not in self._sorted:
            self._sorted[(tag, nbytes)] = R.masked_sorted(self.index[tag][1], nbytes)
        return self._sorted[(tag, nbytes)]

    def device(self):
        return _dev(np.concatenate(self.parts))


def _select_ns(threads):
    return sorted({1, 2, 31, 32, 33, threads - 1, threads, threads + 1, 5000, 1 << 20})


def _ks(n):
    return sorted({k for k in (1, 2, n // 2, n - 1, n) if 1 <= k <= n})


@pytest.mark.parametrize('bits,nbytes', SELECT_WIDTHS)
def test_cta_radix_select(H, bits, nbytes):
    dtype = np.uint32 if bits == 32 else np.uint64
    pool = _KeyPool(dtype, np.random.default_rng(bits * 10 + nbytes))
    queries = {}
    for threads in R.BLOCK_SIZES:
        queries[threads] = [(pool.add(dist, n, k), n, k) for n in _select_ns(threads) for k in _ks(n)
                            for dist in R.DISTRIBUTIONS]
    d_keys = pool.device()
    for threads, qs in queries.items():
        nq = len(qs)
        off = _dev(np.int64([pool.offset(t) for t, _, _ in qs]))
        nk = _dev(np.int32([(n, k) for _, n, k in qs]).reshape(-1))
        out_key = torch.empty(nq * threads, dtype=torch.int32 if bits == 32 else torch.int64, device='cuda')
        out_rank = torch.empty(nq * threads, dtype=torch.int32, device='cuda')
        out_scan = torch.empty_like(out_rank)
        blocks = max(1, nq // 4)                    # each CTA runs about four queries back to back
        _ok(H.cta_h_radix_select(bits, nbytes, threads, blocks, _p(d_keys), _p(off), _p(nk), nq, _p(out_key),
                                 _p(out_rank), _p(out_scan), _st()))
        got_key = _host(out_key, dtype).reshape(nq, threads)
        got_rank = _host(out_rank, np.int32).reshape(nq, threads)
        got_scan = _host(out_scan, np.int32).reshape(nq, threads)
        tid = np.arange(threads)
        for q, (tag, n, k) in enumerate(qs):
            key, rank = R.select_from_sorted(pool.masked_sorted(tag, nbytes), k)
            where = (threads, tag[0], n, k)
            assert (got_key[q] == key).all(), (where, hex(int(got_key[q][0])), hex(int(key)))
            assert (got_rank[q] == rank).all(), (where, got_rank[q][0], rank)
            assert np.array_equal(got_scan[q], tid * rank), where


# ------------------------------------------------------------------------------------------------ cta_smallest_sorted

SMALLEST_KS = [1, 2, 3, 100, 511, 512, 513, 1000, 1023, 1024]


@pytest.mark.parametrize('threads', R.BLOCK_SIZES)
def test_cta_smallest_sorted(H, threads):
    rng = np.random.default_rng(threads)
    arrays, qs = [], []
    big = {n: R.distinct_keys(n, rng) for n in (5120, 166000)}      # 166 000: finalize_kernel's scale
    off = 0
    for k in SMALLEST_KS:
        for n in sorted({k - 1, k, k + 1, 1, 5120, 166000}):
            if n < 1:
                continue
            keys = big[n] if n in big else R.distinct_keys(n, rng)
            arrays.append(keys)
            qs.append((off, n, k, keys))
            off += n
    nq = len(qs)
    d_keys = _dev(np.concatenate(arrays))
    d_off = _dev(np.int64([q[0] for q in qs]))
    d_nk = _dev(np.int32([(n, k) for _, n, k, _ in qs]).reshape(-1))
    out = torch.empty(nq * R.SELECT_CAP, dtype=torch.int64, device='cuda')
    _ok(H.cta_h_smallest_sorted(threads, max(1, nq // 4), _p(d_keys), _p(d_off), _p(d_nk), nq, _p(out), _st()))
    got = _host(out, U64).reshape(nq, R.SELECT_CAP)
    for q, (_, n, k, keys) in enumerate(qs):
        want = R.smallest_sorted(keys, k)
        assert np.array_equal(got[q, :want.size], want), (n, k, np.nonzero(got[q, :want.size] != want)[0][:5])


# ------------------------------------------------------------------------------------------------ sync contract

CONTRACT_CASES = {  # mode of cta_h_contract, (n1, k1, n2, k2)
    'sort': (0, (1024, 0, 1024, 0)),
    'select': (1, (2048, 700, 1500, 3)),
    'smallest_n_le_k': (2, (100, 200, 300, 300)),
    'smallest_n_gt_k': (2, (2048, 700, 1500, 100)),
}


@pytest.mark.parametrize('case', list(CONTRACT_CASES))
@pytest.mark.parametrize('threads', R.BLOCK_SIZES)
def test_cta_helpers_need_no_caller_barrier(H, case, threads):
    """Keys written right before each of two calls and the result read right after, with warp 0 alone reading the whole
    first result ~10 us late: a helper that touches the caller's memory before its first barrier corrupts that read."""
    mode, (n1, k1, n2, k2) = CONTRACT_CASES[case]
    rng = np.random.default_rng(threads + mode)
    in1 = R.distinct_keys(2048, rng)
    in2 = R.distinct_keys(2048, rng)
    d1, d2, d_nk = _dev(in1), _dev(in2), _dev(np.int32([n1, k1, n2, k2]))
    out1 = torch.full((R.SELECT_CAP,), -5, dtype=torch.int64, device='cuda')
    out2 = torch.full_like(out1, -5)
    r1 = torch.full((R.SELECT_CAP,), -5, dtype=torch.int32, device='cuda')
    r2 = torch.full_like(r1, -5)
    _ok(H.cta_h_contract(mode, threads, _p(d1), _p(d2), _p(d_nk), _p(out1), _p(out2), _p(r1), _p(r2), _st()))
    got1, got2 = _host(out1, U64), _host(out2, U64)
    if case == 'sort':
        assert np.array_equal(got1, np.sort(in1[:1024])) and np.array_equal(got2, np.sort(in2[:1024]))
    elif case == 'select':
        for got, rank, keys, n, k in ((got1, r1, in1, n1, k1), (got2, r2, in2, n2, k2)):
            key, rk = R.radix_select(keys[:n], k, 8)
            assert (got[:threads] == key).all() and (_host(rank, np.int32)[:threads] == rk).all()
    else:
        for i, (got, keys, n, k) in enumerate(((got1, in1, n1, k1), (got2, in2, n2, k2))):
            want = R.smallest_sorted(keys[:n], k)
            bad = np.nonzero(got[:want.size] != want)[0]
            assert bad.size == 0, ('call %d' % (i + 1), bad[:8])


# ------------------------------------------------------------------------------------------------ consumers

CHUNK = 1024 * 16                   # pair_select_kernel's compaction chunk: NT threads x PAIR_RUN pairs


def _pair_case(H_img, W_img, level0_logits):
    """Level 0's 80 class logits per pair (pair = location * 80 + class) from level0_logits(n_pairs); every pair of the
    other levels fails the threshold."""
    from test_gpu_benchmark import STRIDES, _pyramid
    sizes = _pyramid(H_img, W_img)
    g = torch.Generator().manual_seed(H_img)
    h0, w0 = sizes[0]
    cls = [torch.from_numpy(np.float32(level0_logits(h0 * w0 * 80)).reshape(h0, w0, 80)).permute(2, 0, 1).contiguous()]
    cls += [torch.full((80, h, w), -6.0) for h, w in sizes[1:]]
    box = [(torch.randn(4, h, w, generator=g) * 4 * s).abs() for (h, w), s in zip(sizes, STRIDES)]
    ctr = [torch.zeros(1, h, w) for h, w in sizes]
    return cls, box, ctr


def test_pair_select_tie_budget_spans_the_chunk_boundary():
    """Pairs below 16 380 fail, every later one has the same score: the 1000 ties taken are pairs 16 380 .. 17 379, four
    in the first chunk and the rest on the tie count carried into the second."""
    from test_gpu_benchmark import _assert_same_candidates, _decode_both

    def logits(n):
        x = np.full(n, 1.0)
        x[:CHUNK - 4] = -6.0
        return x
    cls, box, ctr = _pair_case(128, 256, logits)
    got, want = _decode_both(cls, box, ctr, (128, 256), 1000)
    _assert_same_candidates(got, want)
    assert (got[3] * 80 + got[2]).tolist() == list(range(CHUNK - 4, CHUNK + 996))


def test_pair_select_larger_keys_in_a_later_chunk_than_the_ties():
    """Chunk 0 is all ties, the first 300 pairs of chunk 1 score higher, chunk 2 is ties again: the 300 higher pairs and
    the 700 lowest ties (all in chunk 0), none of chunk 2."""
    from test_gpu_benchmark import _assert_same_candidates, _decode_both

    def logits(n):
        x = np.full(n, -6.0)
        x[:CHUNK] = 1.0
        x[CHUNK:CHUNK + 300] = 2.0
        x[2 * CHUNK:3 * CHUNK] = 1.0
        return x
    cls, box, ctr = _pair_case(256, 320, logits)
    got, want = _decode_both(cls, box, ctr, (256, 320), 1000)
    _assert_same_candidates(got, want)
    assert (got[3] * 80 + got[2]).tolist() == list(range(700)) + list(range(CHUNK, CHUNK + 300))


@pytest.mark.parametrize('num_classes', [1023, 1024])
@pytest.mark.parametrize('max_num', [1, 513, 1024])
def test_multiclass_nms_class_offsets_fill_every_thread(num_classes, max_num):
    """finalize_kernel's class-offset scan with a class per thread (1024) or all but one (1023), more kept boxes than
    max_num, so the cut goes through cta_smallest_sorted."""
    from oracle import ops as O
    from sipmask_b200 import ops
    n = 48
    rng = np.random.default_rng(num_classes + max_num)
    xy = rng.random((n, 2)) * 400
    boxes = torch.from_numpy(np.concatenate([xy, xy + rng.random((n, 2)) * 160 + 1], 1).astype(np.float32))
    # distinct scores above the threshold: every class keeps boxes, and no tie leaves the order to a tie-break
    s = (0.06 + 0.9 * rng.permutation(n * num_classes) / (n * num_classes)).astype(np.float32).reshape(n, num_classes)
    scores = torch.from_numpy(np.concatenate([np.zeros((n, 1), np.float32), s], 1))
    rb, rl, ri = O.multiclass_nms_idx(boxes, scores, 0.05, 0.5, max_num)
    db, dl, di = ops.multiclass_nms_idx(boxes.cuda(), scores.cuda(), 0.05, dict(type='nms', iou_thr=0.5), max_num)
    assert len(ri) == max_num
    assert dl.cpu().tolist() == rl.tolist()
    assert di.cpu().tolist() == ri.tolist()
    np.testing.assert_array_equal(db.cpu().numpy(), rb.numpy())


def test_rle_pack_offsets_at_max_dets():
    """rle_pack_kernel's string offsets with one detection per thread: 1024 and 1023 detections of one image each."""
    from sipmask_b200 import rle
    from test_gpu_rle_stream import _encode
    rng = np.random.default_rng(5)
    N, mx, h, w = 2, 1024, 6, 40
    words = (w + 31) // 32
    counts = [1024, 1023]
    density = rng.random((N, mx, 1, 1))                    # strings of very different lengths
    px = (rng.random((N, mx, h, words * 32)) < density).astype(np.uint8)
    packed = np.packbits(px, axis=-1, bitorder='little').view('<i4').reshape(N, mx, h, words)
    bits = torch.from_numpy(packed.copy()).cuda()
    regions, _ = _encode(bits, torch.tensor(counts, dtype=torch.int32).cuda(), [(h, w)] * N, run_cap=h * w + 2,
                         rle_bytes=1 << 20)
    for i, c in enumerate(counts):
        status, k, strings = rle.read_region(regions[i], mx)
        assert (status, k) == (0, c), i
        assert strings == [rle.encode(px[i, d, :h, :w])['counts'] for d in range(c)], i


@pytest.mark.parametrize('W', [2047, 2048, 2049, 4129])
def test_rle_counts_run_across_the_scan_block_edge(W):
    """rle_counts_kernel scans 2048 columns at a time with a carry: a run that goes from the bottom of the last column
    of a block into the top of the next (or of the last two columns when there is no next), and masks around the
    edge."""
    from oracle import ops as O
    from sipmask_b200 import ops
    h = 5
    rng = np.random.default_rng(W)
    m = np.zeros((6, h, W), np.uint8)
    for c in {min(2047, W - 2), min(4095, W - 2)}:
        m[0, 2:, c] = 1
        m[0, :3, c + 1] = 1
    m[1] = 1
    m[2] = rng.integers(0, 2, (h, W))
    m[3, :, ::2] = 1
    x0 = min(2038, W - 20)
    m[4, :, x0:x0 + 20] = rng.integers(0, 2, (h, 20))
    words = (W + 31) // 32
    pad = np.ones((m.shape[0], h + 2, words * 32), np.uint8)       # junk outside the crop
    pad[:, :h, :W] = m
    bits = np.packbits(pad, axis=-1, bitorder='little').view('<i4').reshape(m.shape[0], h + 2, words)
    bits_t = torch.from_numpy(bits.copy()).cuda()
    counts, n = ops.mask_rle_counts(bits_t, h, W, cap=h * W + 2)
    counts, n = counts.cpu().numpy().view(np.uint32), n.cpu().numpy()
    rles = ops.masks_to_rle(bits_t, h, W, m.shape[0])
    for i in range(m.shape[0]):
        want = O.rle_counts(m[i])
        assert counts[i, :n[i]].tolist() == list(want), i
        assert rles[i]['counts'] == O.rle_to_string(want), i
