"""jsmpeg_b200_batch_write_ps_many on the H100: request i is write_ps on its stream (ES, PES table, host mirror, bytes
left over, in-sync state) and what the serial model (tools/mini_ps.py) gives, for any interleaving with write_ps;
what it ingests decodes bit-exact; streams it does not name are untouched; refusals change nothing; and its launches
grow neither with the number of requests nor with the breaks in the input."""
import ctypes

import numpy as np
import pytest

import helpers
import mini_ps
import ps_cases
from helpers import assert_frames_equal, decode_all
from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder
from ps_many_cases import breaks, candidates, chunked, two_video_program_stream

pytestmark = pytest.mark.gpu

CHUNKS = [None, 1, 64, 333, 2048, 65536, "random"]


def _corpus():
    out = [v[0] for _, v in sorted(ps_cases.TINY.items())]
    for k, name in enumerate(sorted(ps_cases.WRITER)):
        data, _ = ps_cases.writer_case(name)
        out.append(data)
        out.append(ps_cases.damaged(data, ("flips", "lengths", "garbage")[k % 3], 20 + k))
    return out


def _host_mirror(bd, s):
    """The stream's host bit buffer: the write pointer of a 0-byte write, minus the length."""
    length = len(bd.read_es(s))
    ptr = bd.lib.jsmpeg_b200_batch_get_write_ptr(bd.handle, s, 0)
    return ctypes.string_at(ptr - length, length) if length else b""


def _calls(feeds, rng):
    """Calls naming random subsets of the streams that still have pieces, each stream at most once per call."""
    pending = [list(ch) for ch in feeds]
    calls = []
    while any(pending):
        live = [s for s in range(len(feeds)) if pending[s]]
        k = int(rng.integers(1, len(live) + 1))
        calls.append([(int(s), pending[s].pop(0)) for s in rng.permutation(live)[:k]])
    return calls


def test_write_ps_many_equals_write_ps_and_the_model_per_stream():
    rng = np.random.default_rng(1)
    datas = _corpus()
    feeds = [chunked(d, CHUNKS[k % len(CHUNKS)] or len(d), rng) for k, d in enumerate(datas)]
    one, many = BatchDecoder(len(feeds)), BatchDecoder(len(feeds))
    models = [mini_ps.Demuxer() for _ in feeds]
    got_one, got_many = [[] for _ in feeds], [[] for _ in feeds]
    calls = _calls(feeds, rng)
    for c in calls:
        for s, data in c:
            got_one[s].append(one.write_ps(s, data))
            models[s].write(data)
        for (s, _), r in zip(c, many.write_ps_many(c)):
            got_many[s].append(r)
    assert max(len(c) for c in calls) >= 8
    for s in range(len(feeds)):
        assert got_many[s] == got_one[s], f"stream {s}: totals / PES tables"
        es = many.read_es(s)
        assert es == one.read_es(s) == bytes(models[s].es), f"stream {s}: ES"
        assert _host_mirror(many, s) == es == _host_mirror(one, s), f"stream {s}: host mirror"
        assert [(o, round(p * 90000)) for r in got_many[s] for o, p in r[1]] == models[s].pes, f"stream {s}: PES table"
    # the left-over bytes and the in-sync state carry into the next call the same way
    tail = ps_cases.writer_case("mpg_all")[0][:5000]
    for bd in (one, many):
        bd.reset()
    for cut in (5, 2500):
        a = [one.write_ps(s, tail[:cut]) for s in range(2)] + [one.write_ps(s, tail[cut:]) for s in range(2)]
        b = many.write_ps_many([(0, tail[:cut]), (1, tail[:cut])]) + many.write_ps_many([(0, tail[cut:]), (1, tail[cut:])])
        assert a == b and sum(x[0] for x in a) > 0
    one.close()
    many.close()


def test_interleaved_with_write_ps_write_and_write_ts_and_streams_not_named_are_untouched():
    import gen_streams
    from jsmpeg_b200 import ts
    rng = np.random.default_rng(2)
    datas = _corpus()[7:13]
    feeds = [chunked(d, CHUNKS[k % len(CHUNKS)] or len(d), rng) for k, d in enumerate(datas)]
    n = len(feeds)
    bd = BatchDecoder(n + 2)
    models = [mini_ps.Demuxer() for _ in feeds]
    # stream n: a decoded .mpg stream with bytes left over; stream n + 1: write_ts and plain writes; no call names them
    clip = gen_streams.make_clip_ps(176, 144, 6, seed=9)
    bd.write_ps(n, clip[:len(clip) - 3000])
    assert bd.decode(1, OUT_DEVICE)
    before = (bd.read_es(n), bd.get_index(n), bd.read_planes(n))
    tsclip = gen_streams.make_clip_ts(176, 144, 6, seed=10)
    tsparts = chunked(tsclip, 5000)
    for j, c in enumerate(_calls(feeds, rng)):
        if j % 2:
            for s, data in c:
                bd.write_ps(s, data)
        else:
            bd.write_ps_many(c)
        for s, data in c:
            models[s].write(data)
        if j < len(tsparts):
            bd.write_ts(n + 1, tsparts[j])
    for part in tsparts[j + 1:]:
        bd.write_ts(n + 1, part)
    for s in range(n):
        assert bd.read_es(s) == bytes(models[s].es), f"stream {s}"
    assert bd.read_es(n + 1) == b"".join(p for _, p in ts.demux_video_es(tsclip))
    es, index, planes = before
    assert bd.read_es(n) == es and bd.get_index(n) == index
    assert_frames_equal([bd.read_planes(n)], [planes], "stream not named")
    # its held-back bytes are still there: the rest of the clip completes it, through write_ps_many
    whole = mini_ps.demux(clip)[0]
    assert bd.write_ps_many([(n, clip[len(clip) - 3000:])])[0][0] == len(whole) - len(es)
    assert bd.read_es(n) == whole
    bd.close()


@pytest.mark.parametrize("form", ["mpg", "vob"])
def test_ffmpeg_program_streams_ingested_by_write_ps_many_decode_bit_exact(form):
    import gen_streams
    sizes = [(320, 240, 24), (640, 480, 13), (352, 288, 18), (1280, 720, 12)]
    clips = [gen_streams.make_clip_ps(w, h, n, seed=40 + k, form=form) for k, (w, h, n) in enumerate(sizes)]
    m1vs = [gen_streams.make_clip_m1v(w, h, n, seed=40 + k) for k, (w, h, n) in enumerate(sizes)]
    feeds = [chunked(c, size) for c, size in zip(clips, (65536, 16384, 4096, len(clips[3])))]
    bd = BatchDecoder(len(clips))
    for j in range(max(len(f) for f in feeds)):
        bd.write_ps_many([(s, f[j]) for s, f in enumerate(feeds) if j < len(f)])
    exp = [decode_all(helpers.oracle_lib(), [(0, m)]) for m in m1vs]
    for s in range(len(clips)):
        assert bd.read_es(s) == m1vs[s], f"stream {s}"
    n = 0
    while bd.decode(1, OUT_DEVICE):
        for s in range(len(clips)):
            if n < len(exp[s][0]):
                assert_frames_equal([bd.read_planes(s)], [exp[s][0][n]], f"{form} stream {s} picture {n}")
        n += 1
    assert n == max(len(e[0]) for e in exp)
    for s in range(len(clips)):
        assert bd.get_index(s) == exp[s][1][-1]
    for _, _, od in exp:
        od.destroy()
    bd.close()


def test_ipb_clip_with_hostile_audio_decodes_b_pictures_bit_exact():
    import mini_enc
    es = mini_enc.make_b_clip(176, 144, 13)[0]
    data, _ = mini_ps.mux(es, form="mpg", packet=900, audio=600, padding=True, seed=9)
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1)
    try:
        exp_frames, _, od = decode_all(lib, [(0, es)])
    finally:
        lib.oracle_set_decode_b(0)
    bd = BatchDecoder(2, decode_b=True)  # stream 1: the same stream, whole, in the same calls
    pieces = chunked(data, 1000)
    for k, p in enumerate(pieces):
        bd.write_ps_many([(0, p)] + ([(1, data)] if k == 0 else []))
    assert bd.read_es(0) == es == bd.read_es(1)
    n = 0
    while bd.decode(1, OUT_DEVICE):
        for s in (0, 1):
            assert_frames_equal([bd.read_planes(s)], [exp_frames[n]], f"I/P/B in PS: stream {s} picture {n}")
        n += 1
    assert n == len(exp_frames)
    od.destroy()
    bd.close()


def test_two_video_streams_of_one_vob_to_two_streams_in_one_call():
    es_a, es_b = ps_cases.video_es(30000, seed=3), ps_cases.video_es(22000, seed=4)
    mux = two_video_program_stream(es_a, es_b, "vob")
    one, many = BatchDecoder(2), BatchDecoder(2)
    for piece in chunked(mux, 4096):
        r = many.write_ps_many([(0, piece, 0xE0), (1, piece, 0xE1)])
        assert r == [one.write_ps(0, piece, 0xE0), one.write_ps(1, piece, 0xE1)]
    for s, (sid, es) in enumerate(((0xE0, es_a), (0xE1, es_b))):
        assert many.read_es(s) == one.read_es(s) == es
        assert many._pes[s] == one._pes[s] and len(many._pes[s]) >= 5
    one.close()
    many.close()


def _raw(bd, writes, n_max, null=(), sids=None):
    """The C call with its own arrays; `null` names the outputs to pass as NULL."""
    n = len(writes)
    streams = np.array([w[0] for w in writes], np.int32)
    keep = [w[1] for w in writes]
    ptrs = (ctypes.c_char_p * max(n, 1))(*keep)
    sizes = np.array([len(w[1]) for w in writes], np.uint64)
    ids = np.array(sids, np.int32) if sids is not None else None
    appended = np.full(max(n, 1), -7, np.int64)
    n_pes = np.full(max(n, 1), -7, np.int32)
    pts = np.zeros(max(n_max, 1), np.uint64)
    off = np.zeros(max(n_max, 1), np.uint32)
    arg = {"appended": appended.ctypes.data, "pts": pts.ctypes.data, "off": off.ctypes.data, "n_pes": n_pes.ctypes.data}
    for k in null:
        arg[k] = None
    r = bd.lib.jsmpeg_b200_batch_write_ps_many(bd.handle, n, streams.ctypes.data, ctypes.addressof(ptrs), sizes.ctypes.data,
                                               ids.ctypes.data if ids is not None else None, arg["appended"], arg["pts"],
                                               arg["off"], n_max, arg["n_pes"])
    return r, appended[:n], n_pes[:n], pts, off


def test_edges_empty_no_whole_item_null_outputs_and_truncation():
    data = ps_cases.writer_case("mpg_sparse_pts")[0]
    bd, ref = BatchDecoder(3), BatchDecoder(3)
    assert bd.write_ps_many([]) == [] and _raw(bd, [], 0)[0] == 0
    # empty requests and requests holding no whole item: nothing appended, the bytes kept
    assert bd.write_ps_many([(0, b""), (1, data[:10]), (2, data[:30])]) == [(0, [])] * 3
    assert bd.write_ps_many([(1, data[10:3000])]) == [ref.write_ps(1, data[:3000])]
    # NULL outputs
    r, _, _, _, _ = _raw(bd, [(0, data[:6000])], 16, null=("appended", "pts", "off", "n_pes"))
    assert r == ref.write_ps(0, data[:6000])[0] > 0
    # truncation: the first n_max PES table entries in (request, offset) order, n_pes counts them all
    rest0, rest2 = data[6000:], data[30:]
    want0, want2 = ref.write_ps(0, rest0), ref.write_ps(2, data[:30] + rest2)
    assert len(want0[1]) >= 3 and len(want2[1]) >= 3
    n_max = len(want0[1]) + 2
    r, appended, n_pes, pts, off = _raw(bd, [(0, rest0), (2, rest2)], n_max)
    assert r == want0[0] + want2[0] and list(appended) == [want0[0], want2[0]]
    assert list(n_pes) == [len(want0[1]), len(want2[1])]
    table = [(o, round(p * 90000)) for o, p in want0[1] + want2[1]][:n_max]
    assert [(int(o), int(p)) for o, p in zip(off[:n_max], pts[:n_max])] == table
    for s in range(3):
        assert bd.read_es(s) == ref.read_es(s)
    # write_ps with a small n_max keeps the first entries in stream order
    small = BatchDecoder(1)
    pts1, off1, cnt = np.zeros(2, np.uint64), np.zeros(2, np.uint32), ctypes.c_int()
    assert small.lib.jsmpeg_b200_batch_write_ps(small.handle, 0, data, len(data), 0xE0, pts1.ctypes.data, off1.ctypes.data, 2,
                                                ctypes.byref(cnt)) > 0
    full = mini_ps.demux(data)[1]
    assert cnt.value == len(full) and [(int(o), int(p)) for o, p in zip(off1, pts1)] == full[:2]
    for d in (bd, ref, small):
        d.close()


def test_refusals_change_nothing_and_a_dead_batch_answers_minus_one():
    data = ps_cases.writer_case("vob_all")[0]
    bd, clean = BatchDecoder(2), BatchDecoder(2)
    for d in (bd, clean):
        d.write_ps(0, data[:1000])
        d.reset_stats()
    refused = [
        [(0, data[1000:2000]), (0, data[2000:3000])],  # named twice
        [(2, data[1000:2000])],  # out of range
        [(-1, data[1000:2000])],
        [(0, data[1000:2000], 0xC0)],  # not a video stream id
        [(1, data[1000:2000], 0xE1), (0, data[1000:2000], 0xF0)],
    ]
    for writes in refused:
        sids = [w[2] if len(w) > 2 else 0xE0 for w in writes]
        assert _raw(bd, writes, 8, sids=sids)[0] == -2
        with pytest.raises(ValueError):
            bd.write_ps_many(writes)
    streams = np.zeros(1, np.int32)
    ptrs = (ctypes.c_char_p * 1)(None)
    sizes = np.array([10], np.uint64)
    assert bd.lib.jsmpeg_b200_batch_write_ps_many(bd.handle, 1, streams.ctypes.data, ctypes.addressof(ptrs), sizes.ctypes.data,
                                                  None, None, None, None, 0, None) == -2
    assert bd.lib.jsmpeg_b200_batch_write_ps_many(bd.handle, -1, None, None, None, None, None, None, None, 0, None) == -2
    assert bd.lib.jsmpeg_b200_batch_write_ps_many(bd.handle, 1, None, None, None, None, None, None, None, 0, None) == -2
    assert bd.stats() == clean.stats()
    assert bd.read_es(0) == clean.read_es(0) and bd.read_es(1) == clean.read_es(1) == b""
    assert bd.last_error() is None
    assert bd.write_ps_many([(0, data[1000:])]) == clean.write_ps_many([(0, data[1000:])])
    assert bd.read_es(0) == clean.read_es(0) == mini_ps.demux(data)[0]
    bd.close()
    clean.close()
    # a dead batch: -1
    from jsmpeg_b200 import capi
    lib = capi.product_library()
    dead = lib.jsmpeg_b200_batch_create(1, 999, 2)
    assert lib.jsmpeg_b200_batch_last_error(dead)
    streams = np.zeros(1, np.int32)
    ptrs = (ctypes.c_char_p * 1)(data[:500])
    sizes = np.array([500], np.uint64)
    assert lib.jsmpeg_b200_batch_write_ps_many(dead, 1, streams.ctypes.data, ctypes.addressof(ptrs), sizes.ctypes.data, None,
                                               None, None, None, 0, None) == -1
    lib.jsmpeg_b200_batch_destroy(dead)


def _levels(most):
    levels = 1
    while (1 << levels) < most:
        levels += 1
    return levels


def test_launches_grow_neither_with_the_requests_nor_with_the_breaks_and_bytes_are_counted():
    """A call queues 11 + 2 x levels launches (candidates, sort, pack, suffix minimum, link, levels doublings, heads,
    levels + 1 markings, classify, place scan, totals, gather), levels = ceil(log2) of the largest request's candidate
    count; a cub algorithm counts as one launch."""
    clean = ps_cases.writer_case("mpg_all", n=48000)[0]
    cands = candidates(clean)
    damaged = None
    for seed in range(40):
        d = ps_cases.damaged(clean, "lengths", seed)
        if candidates(d) == cands and breaks(d) >= 3:
            damaged = d
            break
    assert damaged is not None and breaks(clean) == 0
    want = 11 + 2 * _levels(cands)
    seen = {}
    for name, data, n in (("clean_1", clean, 1), ("clean_64", clean, 64), ("damaged_1", damaged, 1), ("damaged_64", damaged, 64)):
        bd = BatchDecoder(64)
        bd.reset_stats()
        res = bd.write_ps_many([(s, data) for s in range(n)])
        st = bd.stats()
        assert st["h2d_bytes"] == n * len(data)
        assert st["d2h_bytes"] == sum(a for a, _ in res) > 0
        assert all(r == res[0] for r in res)
        seen[name] = st["kernel_launches"]
        # the staged bytes count once per call: a byte left over is uploaded again with the next call's bytes; plain
        # writes that were not resident yet count when a call appends to their stream
        bd.reset_stats()
        bd.write(0, b"\x00\x00\x01\xb3" + bytes(60))
        r = bd.write_ps_many([(0, clean[:3000]), (1, b"\x00")])
        st = bd.stats()
        assert r[0][0] > 0 and st["h2d_bytes"] == 3000 + 1 + 64 and st["d2h_bytes"] == r[0][0]
        bd.reset_stats()
        bd.write_ps_many([(1, b"\x00\x01")])
        assert bd.stats()["h2d_bytes"] == 3 and bd.stats()["d2h_bytes"] == 0
        bd.close()
    assert seen == {"clean_1": want, "clean_64": want, "damaged_1": want, "damaged_64": want}, seen


def _long_breaks(data, seed, n=40):
    """`data` with runs of random bytes and a false pack-header prefix inserted at n places, and with the
    packet_length of some packets raised to near 64 KB: items that stay incomplete across several 64 KB writes, so
    every call carries tens of KB of left-over bytes into the next."""
    rng = np.random.default_rng(seed)
    b = bytearray(data)
    starts = [i for i in range(len(b) - 6) if b[i:i + 3] == b"\x00\x00\x01" and b[i + 3] > 0xBA]
    for i in rng.choice(starts, min(len(starts), 6), replace=False):
        b[i + 4:i + 6] = int(rng.integers(60000, 65536)).to_bytes(2, "big")
    for at in sorted(rng.integers(0, len(b), n), reverse=True):
        b[at:at] = rng.integers(0, 256, int(rng.integers(1, 300)), dtype=np.uint8).tobytes() + b"\x00\x00\x01\xba"
    return bytes(b)


def test_damaged_program_streams_of_many_streams_in_64_kb_rounds_with_large_left_overs():
    """64 streams of damaged .mpg / .vob, each fed twice over in 64 KB rounds: every call carries left-over bytes (up
    to ~64 KB per stream) into the next.  Byte for byte the same as write_ps and as the model, stream by stream."""
    import gen_streams
    clips = [gen_streams.make_clip_ps(640, 480, 48, seed=300 + k % 8, form=("mpg", "vob")[k % 2]) for k in range(8)]
    datas = [_long_breaks(clips[k % 8], 500 + k) * 2 for k in range(64)]
    pieces = [chunked(d, 65536) for d in datas]
    one, many = BatchDecoder(64), BatchDecoder(64)
    models = [mini_ps.Demuxer() for _ in datas]
    held = 0
    for j in range(max(len(p) for p in pieces)):
        rnd = [(s, p[j]) for s, p in enumerate(pieces) if j < len(p)]
        got = many.write_ps_many(rnd)
        assert got == [one.write_ps(s, data) for s, data in rnd], f"round {j}"
        for s, data in rnd:
            models[s].write(data)
            held = max(held, len(models[s].leftover))
    assert held > 30000
    for s in range(64):
        es = many.read_es(s)
        assert es == one.read_es(s), f"stream {s}: write_ps_many against write_ps"
        assert es == bytes(models[s].es), f"stream {s}: against the model"
        assert _host_mirror(many, s) == es
    assert many.last_error() is None and one.last_error() is None
    one.close()
    many.close()
