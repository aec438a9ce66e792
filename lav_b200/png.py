"""The host half of decoding the recordings' grayscale map PNGs on the device: the chunk walk of each PNG and the packing of a
batch's zlib streams and job table for ops.png_decode_gray8.

parse() checks the signature, that IHDR comes first, every chunk's CRC (a critical chunk with a bad CRC is an error, an
ancillary one is skipped, as libpng does) and concatenates the IDAT payloads.  A plane whose IHDR says 8-bit grayscale, not
interlaced and of the map size goes to the device decoder; any other valid PNG is decoded here by synth.decode_png (cv2), so
every input decodes as cv2.imdecode(..., IMREAD_GRAYSCALE) decodes it."""
import struct
import zlib

import numpy as np

from .capi import LavbError
from .ops import PNG_JOB_DTYPE
from .synth import decode_png

SIGNATURE = b"\x89PNG\r\n\x1a\n"


def chunks(data, what):
    """the (type, payload) chunks of PNG ``data`` up to IEND, CRCs checked; -> (IHDR fields (w, h, depth, color, interlace),
    the concatenated IDAT payloads, the set of chunk types)."""
    def bad(why):
        return LavbError(f"{what}: malformed PNG ({why})")
    data = memoryview(data)
    if len(data) < 8 or bytes(data[:8]) != SIGNATURE:
        raise bad("no PNG signature")
    pos, ihdr, idat, types = 8, None, [], set()
    while True:
        if pos + 8 > len(data):
            raise bad("truncated before IEND")
        n, tag = struct.unpack(">I4s", data[pos:pos + 8])
        if n > 0x7FFFFFFF or pos + 12 + n > len(data):
            raise bad(f"chunk {tag!r} truncated")
        body = data[pos + 8:pos + 8 + n]
        crc = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0]
        critical = not tag[0] & 0x20
        if ihdr is None and tag != b"IHDR":
            raise bad("IHDR is not the first chunk")
        pos += 12 + n
        if zlib.crc32(body, zlib.crc32(tag)) != crc:
            if critical:
                raise bad(f"CRC mismatch in chunk {tag!r}")
            continue
        types.add(tag)
        if tag == b"IHDR":
            if ihdr is not None or n != 13:
                raise bad("bad IHDR")
            w, h, depth, color, comp, filt, interlace = struct.unpack(">IIBBBBB", body)
            if w == 0 or h == 0 or comp != 0 or filt != 0 or interlace > 1:
                raise bad("bad IHDR fields")
            ihdr = (w, h, depth, color, interlace)
        elif tag == b"IDAT":
            idat.append(body)
        elif tag == b"IEND":
            break
    if not idat:
        raise bad("no IDAT chunk")
    return ihdr, b"".join(idat), types


def parse(data, what, size):
    """PNG bytes of a (size, size) plane -> (zlib stream, None) for the device decoder, or (None, plane) decoded on the host for
    any other valid PNG.  Raises LavbError naming ``what`` (trajectory path and key) for a malformed PNG or another size."""
    (w, h, depth, color, interlace), stream, types = chunks(data, what)
    if (h, w) != (size, size):
        raise LavbError(f"{what}: a {h}x{w} PNG where the map size is {size}x{size}")
    if depth == 8 and color == 0 and interlace == 0 and b"tRNS" not in types:
        return stream, None
    plane = decode_png(bytes(data))
    if plane is None or plane.shape != (size, size):
        raise LavbError(f"{what}: the PNG does not decode to a {size}x{size} grayscale plane")
    return None, plane


def pack(parsed, size):
    """the parsed planes of a batch, in plane order -> (uint8 source buffer of the device streams, PNG_JOB_DTYPE job table, list of
    (plane index, host-decoded plane))."""
    streams = [(p, s) for p, (s, _) in enumerate(parsed) if s is not None]
    lens = np.array([len(s) for _, s in streams], np.int64)
    jobs = np.zeros(len(streams), PNG_JOB_DTYPE)
    jobs["off"] = np.concatenate([[0], np.cumsum(lens)[:-1]]) if len(lens) else []
    jobs["len"], jobs["dst"], jobs["h"], jobs["w"] = lens, [p for p, _ in streams], size, size
    src = np.frombuffer(b"".join(s for _, s in streams), np.uint8)
    return src, jobs, [(p, plane) for p, (_, plane) in enumerate(parsed) if plane is not None]
