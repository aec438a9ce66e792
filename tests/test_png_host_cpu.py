"""CPU: the host half of the device PNG decode (lav_b200.png): the chunk walk of the recordings' map PNGs, its errors, the
routing of other PNG kinds to the host decoder, and the packed staging of a batch."""
import struct
import zlib

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from lav_b200 import png, synth  # noqa: E402
from lav_b200.capi import LavbError  # noqa: E402
from lav_b200.datasets import stage_maps  # noqa: E402


def chunk(tag, body):
    return struct.pack(">I", len(body)) + tag + body + struct.pack(">I", zlib.crc32(tag + body) & 0xFFFFFFFF)


def split_chunks(data):
    """(tag, body) of every chunk of a well-formed PNG."""
    pos, out = 8, []
    while pos < len(data):
        n, tag = struct.unpack(">I4s", data[pos:pos + 8])
        out.append((tag, data[pos + 8:pos + 8 + n]))
        pos += 12 + n
    return out


def mask(h, w, seed=0):
    return (np.random.RandomState(seed).rand(h, w) > 0.8).astype(np.uint8) * 255


def test_parse_cv2_map():
    img = mask(320, 320)
    data = synth.encode_png(img)
    (w, h, depth, color, interlace), stream, types = png.chunks(data, "t: map_0_00000")
    assert (w, h, depth, color, interlace) == (320, 320, 8, 0, 0)
    assert stream == b"".join(b for t, b in split_chunks(data) if t == b"IDAT")
    assert len(zlib.decompress(stream)) == 320 * 321
    got, plane = png.parse(data, "t: map_0_00000", 320)
    assert got == stream and plane is None


def test_parse_one_byte_idat_chunks():
    img = mask(320, 320, 1)
    data = synth.encode_png(img)
    parts = split_chunks(data)
    stream = b"".join(b for t, b in parts if t == b"IDAT")
    rebuilt = png.SIGNATURE + chunk(b"IHDR", parts[0][1]) + b"".join(chunk(b"IDAT", stream[k:k + 1]) for k in range(len(stream)))
    rebuilt += chunk(b"IEND", b"")
    assert np.array_equal(cv2.imdecode(np.frombuffer(rebuilt, np.uint8), cv2.IMREAD_GRAYSCALE), img)
    assert png.parse(rebuilt, "k", 320) == (stream, None)


def test_bad_ancillary_crc_is_skipped_like_libpng():
    data = synth.encode_png(mask(320, 320, 2))
    text = chunk(b"tEXt", b"a\x00b")
    bad = text[:-1] + bytes([text[-1] ^ 1])
    data2 = data[:33] + bad + data[33:]
    assert png.parse(data2, "k", 320)[0] == png.parse(data, "k", 320)[0]


@pytest.mark.parametrize("kind", ["crc", "truncated", "no_ihdr", "size", "signature", "no_idat"])
def test_malformed_png_raises_with_key(kind):
    data = synth.encode_png(mask(320, 320, 3))
    what = "/rec/traj_07: map_9_00012"
    if kind == "crc":
        k = data.index(b"IDAT") + 10
        data = data[:k] + bytes([data[k] ^ 0x40]) + data[k + 1:]
    elif kind == "truncated":
        data = data[:len(data) // 2]
    elif kind == "no_ihdr":
        parts = split_chunks(data)
        data = png.SIGNATURE + b"".join(chunk(t, b) for t, b in parts[1:])
    elif kind == "size":
        data = synth.encode_png(mask(160, 320))
    elif kind == "signature":
        data = b"\x89PNX" + data[4:]
    else:
        parts = split_chunks(data)
        data = png.SIGNATURE + b"".join(chunk(t, b) for t, b in parts if t != b"IDAT")
    with pytest.raises(LavbError, match="traj_07: map_9_00012"):
        png.parse(data, what, 320)


@pytest.mark.parametrize("kind", ["color", "16bit", "interlaced"])
def test_other_pngs_go_to_the_host_decoder(kind):
    rs = np.random.RandomState(4)
    if kind == "color":
        img = rs.randint(0, 256, (320, 320, 3), dtype=np.uint8)
    elif kind == "16bit":
        img = rs.randint(0, 65536, (320, 320), dtype=np.uint16)
    else:
        img = None
    if img is not None:
        data = cv2.imencode(".png", img)[1].tobytes()
    else:                                                   # Adam7, written by hand: cv2 does not write interlaced PNGs
        plane = mask(320, 320, 5)
        passes = [(0, 0, 8, 8), (0, 4, 8, 8), (4, 0, 8, 4), (0, 2, 4, 4), (2, 0, 4, 2), (0, 1, 2, 2), (1, 0, 2, 1)]
        raw = b"".join(b"\x00" + plane[y, x0::dx].tobytes() for y0, x0, dy, dx in passes for y in range(y0, 320, dy))
        data = (png.SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", 320, 320, 8, 0, 0, 0, 1)) + chunk(b"IDAT", zlib.compress(raw))
                + chunk(b"IEND", b""))
        assert np.array_equal(cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_GRAYSCALE), plane)
    stream, plane = png.parse(data, "k", 320)
    assert stream is None
    assert np.array_equal(plane, cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_GRAYSCALE))


def test_stage_maps_packs_a_two_sample_batch():
    rs = np.random.RandomState(6)
    imgs = [mask(320, 320, s) for s in range(5)]
    color = rs.randint(0, 256, (320, 320, 3), dtype=np.uint8)
    pngs = [synth.encode_png(i) for i in imgs] + [cv2.imencode(".png", color)[1].tobytes()]
    parsed = [png.parse(d, "k", 320) for d in pngs]
    hs = [dict(pngs=[("map_0_00001", parsed[0]), ("map_9_00001", parsed[5]), ("map_10_00001", parsed[1])]),
          dict(pngs=[("map_0_00004", parsed[2]), ("map_9_00004", parsed[3]), ("map_10_00004", parsed[4])])]
    st = stage_maps(hs, pin=False)
    streams = [parsed[k][0] for k in (0, 1, 2, 3, 4)]
    assert st["n_planes"] == 6 and st["keys"] == ["map_0_00001", "map_9_00001", "map_10_00001", "map_0_00004", "map_9_00004",
                                                  "map_10_00004"]
    assert bytes(st["src"].numpy()) == b"".join(streams)
    jobs = st["jobs"]
    assert jobs.dtype.itemsize == 32 and jobs["dst"].tolist() == [0, 2, 3, 4, 5]
    assert jobs["len"].tolist() == [len(s) for s in streams]
    assert jobs["off"].tolist() == np.concatenate([[0], np.cumsum([len(s) for s in streams])[:-1]]).tolist()
    assert (jobs["h"] == 320).all() and (jobs["w"] == 320).all()
    (p, plane), = st["host"]
    assert p == 1 and np.array_equal(plane.numpy(), cv2.imdecode(np.frombuffer(pngs[5], np.uint8), cv2.IMREAD_GRAYSCALE))
