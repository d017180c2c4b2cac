"""GPU test: every bulk download path yields the same bitmaps at the same indices and reports the
same rb200_last_download_bytes: download_all, the streaming download at several chunk sizes, and
the visitor paths (foreach, foreach_many, foreach_async + download_wait), with visitors that keep
or release the bitmaps.  Results are compared as per-index sha256 digests of their portable
serialization, so host memory stays bounded."""
import ctypes as C
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _digest(rb, p):
    return hashlib.sha256(rb.Bitmap(p, own=False).serialize()).digest()


def _visitor(rb, n, keep):
    """visit(index, bitmap) recording the bitmap's digest; keep=True takes ownership (returns 1)
    and frees the bitmap itself."""
    digs = [None] * n

    def visit(i, p):
        digs[i] = _digest(rb, p)
        if keep:
            rb.Bitmap(p).free()
        return 1 if keep else 0
    return visit, digs


def _c_visitor(rb, visit):
    return rb.api.VISIT_FN(lambda i, p, _ctx: visit(i, p))


def _all_paths(rb, S):
    """path -> (per-index digests, rb200_last_download_bytes right after the path ran)."""
    lib = rb.api.lib()
    n = len(S)
    got, chunks = {}, {}
    arr = S.download_all_raw()
    got["download_all"] = ([_digest(rb, arr[i]) for i in range(n)], lib.rb200_last_download_bytes())
    S.free_raw(arr)
    for cb in (1, 97, 4096, None):
        digs, chunks[cb] = [], 0
        for a, m in (S.download_stream(cb) if cb else S.download_stream()):
            assert 0 < m <= (cb or 1024)
            digs += [_digest(rb, a[k]) for k in range(m)]
            S.free_raw(a, m)
            chunks[cb] += 1
        got[f"download_stream({cb})"] = (digs, lib.rb200_last_download_bytes())
    for keep in (False, True):
        visit, digs = _visitor(rb, n, keep)
        fn = _c_visitor(rb, visit)
        assert lib.rb200_download_foreach(S.ptr, C.cast(fn, C.c_void_p), None) == 0, rb.last_error()
        got[f"foreach(keep={keep})"] = (digs, lib.rb200_last_download_bytes())
        visit, digs = _visitor(rb, n, keep)
        rb.foreach_many([S], visit)
        got[f"foreach_many(keep={keep})"] = (digs, lib.rb200_last_download_bytes())
        visit, digs = _visitor(rb, n, keep)
        fn = _c_visitor(rb, visit)
        S.foreach_async(None, fn)
        rb.download_wait()
        got[f"foreach_async(keep={keep})"] = (digs, lib.rb200_last_download_bytes())
    return got, chunks


def _check_paths_agree(rb, S):
    got, chunks = _all_paths(rb, S)
    ref_digs, ref_bytes = got["download_all"]
    assert len(ref_digs) == len(S)
    for path, (digs, nbytes) in got.items():
        assert digs == ref_digs, path
        assert nbytes == ref_bytes, path
    return ref_digs, ref_bytes, chunks


def test_many_sets_and_queued_jobs(rb):
    """foreach_many over [small, empty, large] numbers the bitmaps across the sets; foreach_async
    with a small job queued before a larger one grows the downloader's ring between the jobs (when
    this is the process's first asynchronous download, as it is when this file runs alone or first
    of the visitor tests)."""
    lib = rb.api.lib()
    blobs = rb.load_realdata("weather_sept_85")
    S = rb.DeviceSet.from_serialized(blobs)
    small = S.batch("and", S, np.arange(30, dtype=np.uint32), np.arange(1, 31, dtype=np.uint32))
    empty = S.batch("and", S, np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    i, j = np.triu_indices(len(blobs), 1)
    large = S.batch("xor", S, i.astype(np.uint32), j.astype(np.uint32))
    ref, ref_bytes = [], []
    for s in (small, empty, large):
        arr = s.download_all_raw()
        ref.append([_digest(rb, arr[k]) for k in range(len(s))])
        ref_bytes.append(lib.rb200_last_download_bytes())
        s.free_raw(arr)
    for keep in (False, True):
        visit, digs = _visitor(rb, len(small) + len(large), keep)
        rb.foreach_many([small, empty, large], visit)
        assert digs == ref[0] + ref[2]
        assert lib.rb200_last_download_bytes() == sum(ref_bytes)
    # small first: the ring is sized for it, then must grow (with nothing in flight) for `large`
    visitors = [_visitor(rb, len(s), keep=False) for s in (small, empty, large)]
    fns = [_c_visitor(rb, visit) for visit, _ in visitors]
    for s, fn in zip((small, empty, large), fns):
        s.foreach_async(None, fn)
    rb.download_wait()
    assert [digs for _, digs in visitors] == ref
    assert lib.rb200_last_download_bytes() == sum(ref_bytes)


@pytest.mark.parametrize("bound", [False, True])
def test_all_pairs_or_paths_agree(rb, R, bound):
    blobs = rb.load_realdata("weather_sept_85")
    host = [rb.Bitmap.deserialize(b) for b in blobs]
    S = rb.DeviceSet.upload(host).bind_host() if bound else rb.DeviceSet.from_serialized(blobs)
    i, j = np.triu_indices(len(blobs), 1)
    assert len(i) == 19900
    res = S.batch("or", S, i.astype(np.uint32), j.astype(np.uint32))
    digs, nbytes, chunks = _check_paths_agree(rb, res)
    # the visitor paths cut chunks of <= 4096 bitmaps: more chunks than their 4 staging slots, and
    # far more than download_stream's 2, so both rings wrap
    assert chunks[4096] >= 5 and chunks[None] >= 20 and chunks[1] == len(i)
    assert nbytes > 0
    for k in range(0, len(i), 997):
        assert digs[k] == hashlib.sha256(R.op_bytes("or", blobs[i[k]], blobs[j[k]])).digest(), k


def test_empty_bitmaps_and_empty_set(rb, R):
    blobs = rb.load_realdata("weather_sept_85")[:40]
    S = rb.DeviceSet.from_serialized(blobs)
    ia = np.arange(40, dtype=np.uint32)
    ib = np.where(ia % 3 == 0, ia, (ia + 1) % 40).astype(np.uint32)   # x ^ x: every third is empty
    res = S.batch("xor", S, ia, ib)
    digs, _, _ = _check_paths_agree(rb, res)
    empty = hashlib.sha256(R.op_bytes("xor", blobs[0], blobs[0])).digest()
    for k in range(40):
        exp = R.op_bytes("xor", blobs[ia[k]], blobs[ib[k]])
        assert digs[k] == hashlib.sha256(exp).digest(), k
        if k % 3 == 0:
            assert digs[k] == empty, k
    assert any(d != empty for d in digs)
    e = S.batch("and", S, np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    digs, nbytes, chunks = _check_paths_agree(rb, e)
    assert digs == [] and nbytes == 0 and all(c == 0 for c in chunks.values())
