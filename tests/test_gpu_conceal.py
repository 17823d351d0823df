"""The `conceal` option on the device (include/jsmpeg_b200.h, DESIGN 3.19) against the rule's model
(tools/conceal_model.py) on the damaged corpus of tests/test_conceal_oracle.py: decode(1) picture by picture (device
planes, host ring, RGBA) with decode_b off and on, the reference ABI through MPEG1Video(concealErrors), decode_frames in
coded and display order, seek_pictures and decode_pictures against the device's own fresh decoder, clean streams
(same bytes, same launches) and the records' exports, which the option leaves as they are."""
import numpy as np
import pytest

import chain_model
import conceal_model
import display_model
import helpers
import intra_model
import synth_es
from jsmpeg_b200 import decoder
from jsmpeg_b200.batch import OUT_ACCUMULATED, OUT_HOST, OUT_MACROBLOCKS, OUT_RESIDUALS, OUT_RGBA, BatchDecoder
from test_conceal_oracle import CORPUS, END, corpus_stream
from test_gpu_intra import ffmpeg_es

pytestmark = pytest.mark.gpu


def model(name, conceal, decode_b):
    return list(conceal_model.decode(helpers.oracle_lib(), corpus_stream(name), conceal, decode_b=decode_b))


def rgba_of(planes, width, height, coded_width):
    """The reference's YCbCr -> RGBA (canvas2d.js) of Y | Cr | Cb: the even part of the display size, the odd edge
    opaque white"""
    ysize = planes.size * 2 // 3
    y = planes[:ysize].reshape(-1, coded_width).astype(np.int32)
    cr = planes[ysize:ysize * 5 // 4].reshape(-1, coded_width // 2).astype(np.int32)
    cb = planes[ysize * 5 // 4:].reshape(-1, coded_width // 2).astype(np.int32)
    h2, w2 = (height >> 1) * 2, (width >> 1) * 2
    yy = y[:h2, :w2]
    cr = np.repeat(np.repeat(cr[:h2 // 2, :w2 // 2], 2, 0), 2, 1)
    cb = np.repeat(np.repeat(cb[:h2 // 2, :w2 // 2], 2, 0), 2, 1)
    r = (cr + ((cr * 103) >> 8)) - 179
    g = ((cb * 88) >> 8) - 44 + ((cr * 183) >> 8) - 91
    b = (cb + ((cb * 198) >> 8)) - 227
    out = np.full((height, width, 4), 255, np.uint8)
    out[:h2, :w2, 0] = np.clip(yy + r, 0, 255)
    out[:h2, :w2, 1] = np.clip(yy - g, 0, 255)
    out[:h2, :w2, 2] = np.clip(yy + b, 0, 255)
    return out


@pytest.mark.parametrize("decode_b", [0, 1])
@pytest.mark.parametrize("name", CORPUS)
def test_every_decode_equals_the_model(name, decode_b):
    es = corpus_stream(name)
    want = model(name, True, decode_b)
    bd = BatchDecoder(1, decode_b=decode_b, conceal=1)
    bd.write(0, es)
    info = bd.stream_info(0)
    for k, p in enumerate(want):
        assert bd.decode(1, OUT_HOST | OUT_RGBA) == 1, (name, k)
        planes = np.concatenate(bd.read_planes(0))
        assert np.array_equal(planes, p["planes"]), (name, k, p["type"])
        assert np.array_equal(np.concatenate([np.array(v) for v in bd.host_planes(0)]), p["planes"]), (name, k, "host")
        if p["decoded"]:
            assert np.array_equal(bd.read_rgba(0), rgba_of(p["planes"], info["width"], info["height"], coded_width(es))), \
                (name, k, "rgba")
    assert bd.last_error() is None
    bd.close()
    # the reference ABI
    v = decoder.MPEG1Video({"decodeFirstFrame": False, "concealErrors": True, "decodeBPictures": bool(decode_b)})
    rec = decoder.PlaneRecorder()
    v.connect(rec)
    v.write(0, [es])
    while v.decode():
        pass
    v.destroy()
    got = [np.concatenate([np.ascontiguousarray(x).reshape(-1) for x in f]) for f in rec.frames]
    assert len(got) == len(want)
    for k, (g, p) in enumerate(zip(got, want)):
        assert np.array_equal(g, p["planes"]), (name, k, "MPEG1Video")


def coded_width(es):
    """the coded width of `es`'s first sequence header (horizontal_size rounded up to whole macroblocks)"""
    h = intra_model.first_sequence_header(es)[0]
    return ((es[h + 4] << 4 | es[h + 5] >> 4) + 15) >> 4 << 4


@pytest.mark.parametrize("decode_b", [0, 1])
@pytest.mark.parametrize("name", ["ip_flips_1", "b_flips_1", "b_clip_flips", "ip_cuts_1"])
def test_decode_frames_equal_the_decode_pictures(name, decode_b):
    es = corpus_stream(name)
    want = [p for p in model(name, True, decode_b) if p["decoded"]]
    n = len(list(model(name, True, decode_b)))
    bd = BatchDecoder(1, decode_b=decode_b, conceal=1)
    bd.write(0, es)
    got = bd.decode_frames(n, rgba=True)[0]
    info = bd.stream_info(0)
    assert got["n_frames"] == len(want)
    for j, p in enumerate(want):
        assert np.array_equal(got["planes"][j].cpu().numpy(), p["planes"]), (name, j)
        assert np.array_equal(got["rgba"][j].cpu().numpy(), rgba_of(p["planes"], info["width"], info["height"],
                                                                    coded_width(es))), (name, j, "rgba")
    bd.close()
    bd = BatchDecoder(1, decode_b=decode_b, conceal=1)
    bd.write(0, es)
    half = n // 2
    shown = []
    for call in (half, n - half):
        r = bd.decode_frames(call, display_order=True)[0]
        shown += [(i["type"], r["planes"][j].cpu().numpy()) for j, i in enumerate(r["info"])]
    r = bd.flush_frames()[0]
    shown += [(i["type"], r["planes"][j].cpu().numpy()) for j, i in enumerate(r["info"])]
    frames = [{"type": p["type"], "planes": p["planes"]} for p in want]
    calls = display_model.present(frames, [len([p for p in list(model(name, True, decode_b))[:half] if p["decoded"]]),
                                           len(frames)], decode_b=bool(decode_b))
    expect = [f for c in calls for f in c]
    assert len(shown) == len(expect)
    for j, ((t, g), f) in enumerate(zip(shown, expect)):
        assert t == f["type"] and np.array_equal(g, f["planes"]), (name, j, "display order")
    bd.close()


def fresh_concealed(data, target, decode_b):
    """(status, Y | Cr | Cb) of the device's own fresh decoder with conceal fed `data`, after it consumes the picture
    whose start code is at byte `target` of `data` (status 0 and zero planes when it never does)"""
    starts = chain_model.picture_positions(data)
    bd = BatchDecoder(1, decode_b=decode_b, conceal=1)
    bd.write(0, data)
    try:
        while True:
            at = (bd.get_index(0) + 7) >> 3
            nxt = next((p for p in starts if p >= at), None)
            if nxt is None or nxt > target:
                return 0, np.zeros(bd.stream_info(0)["coded_size"] * 3 // 2, np.uint8)
            assert bd.decode(1) == 1
            if nxt == target:
                return 1, np.concatenate(bd.read_planes(0))
    finally:
        bd.close()


@pytest.mark.parametrize("name,decode_b", [("ip_flips_1", 0), ("ip_cuts_1", 0), ("b_flips_1", 1), ("b_clip_flips", 1)])
def test_random_access_equals_the_fresh_decoder(name, decode_b):
    """decode_pictures against the fresh decoder fed the chain start and the rest of the buffer (a damaged walk may run
    across the closing code); seek_pictures against the one fed its seek chain start (chain_model.seek_bytes)"""
    es = corpus_stream(name)
    entries = chain_model.picture_index(es, bool(decode_b))
    bd = BatchDecoder(1, decode_b=decode_b, conceal=1)
    bd.write(0, es)
    got = bd.decode_pictures([(0, e["picture"]) for e in entries])
    for e, t, i in zip(entries, got, bd.last_pictures_info):
        data = chain_model.fresh_bytes(es, dict(e, close=len(es) - 4))
        status, planes = fresh_concealed(data, chain_model.target_start_byte(es, e) - 4, decode_b)
        assert i["status"] == status and np.array_equal(t.cpu().numpy(), planes), (name, e["picture"], "decode_pictures")
    for e in entries:
        data = chain_model.seek_bytes(es, e, bool(decode_b))
        status, planes = fresh_concealed(data, e["byte_pos"] - (len(es) - len(data)), decode_b)
        assert bd.seek_pictures([(0, e["picture"])]) == 1
        assert bd.last_seek_info[0]["status"] == status, (name, e["picture"], "seek")
        if status:
            assert np.array_equal(np.concatenate(bd.read_planes(0)), planes), (name, e["picture"], "seek")
    assert bd.last_error() is None
    bd.close()


def run_decodes(es, decode_b, conceal, flags=OUT_HOST | OUT_RGBA, read=None):
    bd = BatchDecoder(1, decode_b=decode_b, conceal=conceal)
    bd.write(0, es)
    out = []
    while bd.decode(1, flags):
        out.append(read(bd) if read else np.concatenate(bd.read_planes(0)))
    launches = bd.stats()["kernel_launches"]
    bd.close()
    return out, launches


@pytest.mark.parametrize("what,decode_b", [("ffmpeg", 0), ("b_one_slice_fcodes", 1), ("b_rows", 1)])
def test_clean_streams_cost_nothing(what, decode_b):
    es = ffmpeg_es(320, 240, 12) + END if what == "ffmpeg" else synth_es.make_case(what)
    off, launches_off = run_decodes(es, decode_b, 0)
    on, launches_on = run_decodes(es, decode_b, 1)
    assert len(on) == len(off) > 0 and launches_on == launches_off
    assert all(np.array_equal(a, b) for a, b in zip(on, off))


def _records(bd):
    return bd.read_macroblocks(0).copy(), bd.read_residuals(0).copy(), bd.read_accumulated(0).copy()


@pytest.mark.parametrize("decode_b", [0, 1])
@pytest.mark.parametrize("name", ["ip_flips_2", "ip_cuts_2", "b_flips_2"])
def test_exports_do_not_change(name, decode_b):
    es = corpus_stream(name)
    flags = OUT_MACROBLOCKS | OUT_RESIDUALS | OUT_ACCUMULATED
    off, launches_off = run_decodes(es, decode_b, 0, flags, _records)
    on, launches_on = run_decodes(es, decode_b, 1, flags, _records)
    assert len(on) == len(off) > 0
    for k, (a, b) in enumerate(zip(on, off)):
        for kind, x, y in zip(("entries", "residuals", "maps"), a, b):
            assert np.array_equal(x, y), (name, k, kind)
    assert launches_on > launches_off  # (the damaged pictures' copies)


def test_concealment_changes_damaged_output():
    differ = 0
    for name in ("ip_flips_1", "ip_cuts_1", "b_clip_flips"):
        decode_b = int(name.startswith("b"))
        es = corpus_stream(name)
        on, _ = run_decodes(es, decode_b, 1)
        off, _ = run_decodes(es, decode_b, 0)
        differ += sum(not np.array_equal(a, b) for a, b in zip(on, off))
    assert differ > 0
