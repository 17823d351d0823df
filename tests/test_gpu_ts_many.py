"""jsmpeg_b200_batch_write_ts_many on the H100: request i is write_ts on its stream (ES, PES table, host mirror, bytes
left over), for any interleaving with write_ts; what it ingests decodes bit-exact; streams it does not name are
untouched; refusals change nothing; and its launches do not grow with the number of requests."""
import ctypes

import numpy as np
import pytest

import ts_many_cases as cases
from helpers import assert_frames_equal, decode_all, oracle_lib
from jsmpeg_b200 import ts
from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder

pytestmark = pytest.mark.gpu

CHUNKS = [None, 188 * 7, 1000, 333, "random"]


def _feeds(n=16, rebind=True):
    """n streams: different clips, sizes and chunkings; garbage on some, and re-binding (which drops PES packets)."""
    import gen_streams
    rng = np.random.default_rng(3)
    feeds = []
    for k in range(n):
        w, h = [(176, 144), (320, 240)][k % 2]
        data = gen_streams.make_clip_ts(w, h, 6 + k % 5, seed=100 + k, noise=4)
        if k % 4 == 1:
            data = cases.with_garbage(data, k)
        if k % 4 == 2 and rebind:
            data = cases.rebound(data, 1, 2)
        chunk = CHUNKS[k % len(CHUNKS)]
        feeds.append((data, cases.chunked(data, chunk or len(data), rng)))
    return feeds


def _host_mirror(bd, s):
    """The stream's host bit buffer: the write pointer of a 0-byte write, minus the length."""
    length = len(bd.read_es(s))
    ptr = bd.lib.jsmpeg_b200_batch_get_write_ptr(bd.handle, s, 0)
    return ctypes.string_at(ptr - length, length) if length else b""


def _rounds(feeds):
    """Round j: the j-th chunk of every stream that still has one."""
    return [[(s, ch[j]) for s, (_, ch) in enumerate(feeds) if j < len(ch)] for j in range(max(len(ch) for _, ch in feeds))]


def test_write_ts_many_equals_write_ts_per_stream():
    feeds = _feeds()
    one, many = BatchDecoder(len(feeds)), BatchDecoder(len(feeds))
    models = [cases.StreamModel() for _ in feeds]
    got_one, got_many = [[] for _ in feeds], [[] for _ in feeds]
    for rnd in _rounds(feeds):
        for s, data in rnd:
            got_one[s].append(one.write_ts(s, data))
            models[s].write(data)
        for (s, _), r in zip(rnd, many.write_ts_many(rnd)):
            got_many[s].append(r)
    for s in range(len(feeds)):
        assert got_many[s] == got_one[s], f"stream {s}: totals / PES tables"
        es = many.read_es(s)
        assert es == one.read_es(s) == models[s].es(), f"stream {s}: ES"
        assert _host_mirror(many, s) == es == _host_mirror(one, s), f"stream {s}: host mirror"
        assert [(o, round(p * 90000)) for r in got_many[s] for o, p in r[1]] == models[s].table
    # the left-over bytes carry into the next call the same way: a packet cut in two, its halves in two calls
    tail = feeds[0][0][:188 * 20 + 100]
    for bd in (one, many):
        bd.reset()
    a = [one.write_ts(s, tail[:288]) for s in range(2)] + [one.write_ts(s, tail[288:]) for s in range(2)]
    b = many.write_ts_many([(0, tail[:288]), (1, tail[:288])]) + many.write_ts_many([(0, tail[288:]), (1, tail[288:])])
    assert a == b and sum(x[0] for x in a) > 0
    one.close()
    many.close()


def test_streams_ingested_by_write_ts_many_decode_bit_exact():
    feeds = _feeds(8, rebind=False)
    bd = BatchDecoder(len(feeds))
    for rnd in _rounds(feeds):
        bd.write_ts_many(rnd)
    exp = []
    for data, _ in feeds:
        exp.append(decode_all(oracle_lib(), ts.demux_video_es(data)))
    n = 0
    while bd.decode(1, OUT_DEVICE):
        for s in range(len(feeds)):
            if n < len(exp[s][0]):
                assert_frames_equal([bd.read_planes(s)], [exp[s][0][n]], f"stream {s} picture {n}")
        n += 1
    assert n == max(len(e[0]) for e in exp) and n >= 6
    for _, _, od in exp:
        od.destroy()
    bd.close()


def test_interleaved_with_write_ts_and_streams_not_named_are_untouched():
    feeds = _feeds(6)
    bd = BatchDecoder(len(feeds) + 1)
    models = [cases.StreamModel() for _ in feeds]
    # stream 6: a decoded stream with bytes left over; no call below names it
    import gen_streams
    other = gen_streams.make_clip_ts(176, 144, 6, seed=9, noise=4)
    bd.write_ts(6, other[:len(other) - 100])
    assert bd.decode(1, OUT_DEVICE)
    before = (bd.read_es(6), bd.get_index(6), bd.read_planes(6))
    for j, rnd in enumerate(_rounds(feeds)):
        if j % 2:
            for s, data in rnd:
                bd.write_ts(s, data)
        else:
            bd.write_ts_many(rnd)
        for s, data in rnd:
            models[s].write(data)
    for s in range(len(feeds)):
        assert bd.read_es(s) == models[s].es(), f"stream {s}"
    es, index, planes = before
    assert bd.read_es(6) == es and bd.get_index(6) == index
    assert_frames_equal([bd.read_planes(6)], [planes], "stream not named")
    # its 100 held-back bytes are still there: the rest of the clip completes it
    whole = b"".join(p for _, p in ts.demux_video_es(other))
    assert bd.write_ts(6, other[len(other) - 100:])[0] == len(whole) - len(es)
    assert bd.read_es(6) == whole
    bd.close()


def test_two_programs_of_one_multiplex():
    import gen_streams
    a = gen_streams.make_clip_ts(176, 144, 8, seed=31, noise=4)
    b = gen_streams.make_clip_ts(320, 240, 8, seed=32, noise=4)
    mux = cases.two_programs(a, b)
    one, many = BatchDecoder(2), BatchDecoder(2)
    for piece in cases.chunked(mux, 4096):
        r = many.write_ts_many([(0, piece, 0xE0), (1, piece, 0xE1)])
        assert r == [one.write_ts(0, piece, 0xE0), one.write_ts(1, piece, 0xE1)]
    for s, clip in ((0, a), (1, b)):
        assert many.read_es(s) == one.read_es(s) == b"".join(p for _, p in ts.demux_video_es(clip))
    exp = [decode_all(oracle_lib(), ts.demux_video_es(c)) for c in (a, b)]
    n = 0
    while many.decode(1, OUT_DEVICE):
        for s in range(2):
            assert_frames_equal([many.read_planes(s)], [exp[s][0][n]], f"program {s} picture {n}")
        n += 1
    assert n == len(exp[0][0]) == len(exp[1][0])
    for _, _, od in exp:
        od.destroy()
    one.close()
    many.close()


def _raw(bd, writes, n_max, null=()):
    """The C call with its own arrays; `null` names the outputs to pass as NULL."""
    n = len(writes)
    streams = np.array([w[0] for w in writes], np.int32)
    keep = [w[1] for w in writes]
    ptrs = (ctypes.c_char_p * max(n, 1))(*keep)
    sizes = np.array([len(w[1]) for w in writes], np.uint64)
    appended = np.full(max(n, 1), -7, np.int64)
    n_pes = np.full(max(n, 1), -7, np.int32)
    pts = np.zeros(max(n_max, 1), np.uint64)
    off = np.zeros(max(n_max, 1), np.uint32)
    arg = {"appended": appended.ctypes.data, "pts": pts.ctypes.data, "off": off.ctypes.data, "n_pes": n_pes.ctypes.data}
    for k in null:
        arg[k] = None
    r = bd.lib.jsmpeg_b200_batch_write_ts_many(bd.handle, n, streams.ctypes.data, ctypes.addressof(ptrs), sizes.ctypes.data,
                                               None, arg["appended"], arg["pts"], arg["off"], n_max, arg["n_pes"])
    return r, appended[:n], n_pes[:n], pts, off


def test_edges_empty_small_null_outputs_and_truncation():
    import gen_streams
    clip = gen_streams.make_clip_ts(176, 144, 10, seed=5, noise=4)
    bd, ref = BatchDecoder(3), BatchDecoder(3)
    assert bd.write_ts_many([]) == [] and _raw(bd, [], 0)[0] == 0
    # empty and sub-packet buffers: nothing appended, the bytes kept
    assert bd.write_ts_many([(0, b""), (1, clip[:100]), (2, clip[:187])]) == [(0, [])] * 3
    assert bd.write_ts_many([(1, clip[100:188 * 4])]) == [ref.write_ts(1, clip[:188 * 4])]
    # NULL outputs
    r, _, _, _, _ = _raw(bd, [(0, clip[:188 * 8])], 16, null=("appended", "pts", "off", "n_pes"))
    assert r == ref.write_ts(0, clip[:188 * 8])[0] > 0
    # truncation: the first n_max PES starts in (request, offset) order, n_pes counts them all
    rest0, rest2 = clip[188 * 8:], clip[187:]
    want0, want2 = ref.write_ts(0, rest0), ref.write_ts(2, clip[:187] + rest2)
    assert len(want0[1]) >= 3 and len(want2[1]) >= 3
    n_max = len(want0[1]) + 1
    r, appended, n_pes, pts, off = _raw(bd, [(0, rest0), (2, rest2)], n_max)
    assert r == want0[0] + want2[0] and list(appended) == [want0[0], want2[0]]
    assert list(n_pes) == [len(want0[1]), len(want2[1])]
    table = [(o, round(p * 90000)) for o, p in want0[1] + want2[1]][:n_max]
    assert [(int(o), int(p)) for o, p in zip(off[:n_max], pts[:n_max])] == table
    # write_ts with a small n_max keeps the first entries in stream order
    small = BatchDecoder(1)
    pts1, off1, cnt = np.zeros(2, np.uint64), np.zeros(2, np.uint32), ctypes.c_int()
    assert small.lib.jsmpeg_b200_batch_write_ts(small.handle, 0, clip, len(clip), 0xE0, pts1.ctypes.data, off1.ctypes.data, 2,
                                                ctypes.byref(cnt)) > 0
    full = ts.demux_video_es(clip)
    assert cnt.value == len(full) and list(off1) == [0, len(full[0][1])]
    for d in (bd, ref, small):
        d.close()


def test_refusals_change_nothing_and_a_dead_batch_answers_minus_one():
    import gen_streams
    clip = gen_streams.make_clip_ts(176, 144, 6, seed=6, noise=4)
    bd, clean = BatchDecoder(2), BatchDecoder(2)
    for d in (bd, clean):
        d.write_ts(0, clip[:1000])
        d.reset_stats()
    refused = [
        [(0, clip[1000:2000]), (0, clip[2000:3000])],  # named twice
        [(2, clip[1000:2000])],  # out of range
        [(-1, clip[1000:2000])],
    ]
    for writes in refused:
        assert _raw(bd, writes, 8)[0] == -2
        with pytest.raises(ValueError):
            bd.write_ts_many(writes)
    streams = np.zeros(1, np.int32)
    ptrs = (ctypes.c_char_p * 1)(None)
    sizes = np.array([10], np.uint64)
    assert bd.lib.jsmpeg_b200_batch_write_ts_many(bd.handle, 1, streams.ctypes.data, ctypes.addressof(ptrs), sizes.ctypes.data,
                                                  None, None, None, None, 0, None) == -2
    assert bd.lib.jsmpeg_b200_batch_write_ts_many(bd.handle, -1, None, None, None, None, None, None, None, 0, None) == -2
    assert bd.stats() == clean.stats()
    assert bd.read_es(0) == clean.read_es(0)
    assert bd.write_ts_many([(0, clip[1000:])]) == clean.write_ts_many([(0, clip[1000:])])
    assert bd.read_es(0) == clean.read_es(0)
    bd.close()
    clean.close()
    # a dead batch: -1
    from jsmpeg_b200 import capi
    lib = capi.product_library()
    dead = lib.jsmpeg_b200_batch_create(1, 999, 2)
    assert lib.jsmpeg_b200_batch_last_error(dead)
    streams = np.zeros(1, np.int32)
    ptrs = (ctypes.c_char_p * 1)(clip[:376])
    sizes = np.array([376], np.uint64)
    assert lib.jsmpeg_b200_batch_write_ts_many(dead, 1, streams.ctypes.data, ctypes.addressof(ptrs), sizes.ctypes.data, None,
                                               None, None, None, 0, None) == -1
    lib.jsmpeg_b200_batch_destroy(dead)


def test_launches_do_not_grow_with_the_requests_and_bytes_are_counted():
    import gen_streams
    clips = [gen_streams.make_clip_ts(176, 144, 6, seed=200 + k, noise=4) for k in range(4)]
    chunk = 188 * 40
    seen = []
    for n in (1, 64):
        bd = BatchDecoder(64)
        writes = [(s, clips[s % 4][:chunk]) for s in range(n)]
        bd.reset_stats()
        res = bd.write_ts_many(writes)
        st = bd.stats()
        assert st["h2d_bytes"] == n * chunk
        assert st["d2h_bytes"] == sum(a for a, _ in res) > 0
        seen.append(st["kernel_launches"])
        bd.close()
    assert seen[0] == seen[1] > 0
