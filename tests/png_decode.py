"""A small PNG reader for the tests of nerfshop_b200/slices.py: checks every chunk's CRC, inflates IDAT with zlib and undoes the five
row filters of 8-bit grey (colour type 0) and RGBA (colour type 6) images. Returns uint8 [h, w] or [h, w, 4]."""
import struct
import zlib

import numpy as np


def decode_png(data: bytes) -> np.ndarray:
    assert data[:8] == b"\x89PNG\r\n\x1a\n", "not a PNG signature"
    pos, idat, hdr, ended = 8, b"", None, False
    while pos < len(data):
        (n,) = struct.unpack(">I", data[pos:pos + 4])
        tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        (crc,) = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        assert zlib.crc32(tag + body) & 0xFFFFFFFF == crc, f"bad CRC in {tag!r}"
        if tag == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", body)
        elif tag == b"IDAT":
            idat += body
        elif tag == b"IEND":
            ended = True
        pos += 12 + n
    assert hdr is not None and ended and pos == len(data)
    w, h, depth, ctype, comp, filt, interlace = hdr
    assert depth == 8 and ctype in (0, 6) and comp == 0 and filt == 0 and interlace == 0
    ch = 1 if ctype == 0 else 4
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + w * ch)
    out = np.zeros((h, w * ch), np.int32)
    for y in range(h):
        f, line = raw[y, 0], raw[y, 1:].astype(np.int32)
        if f == 0:
            out[y] = line
            continue
        prev = out[y - 1] if y else np.zeros(w * ch, np.int32)
        cur = np.zeros(w * ch, np.int32)
        for i in range(w * ch):
            a = cur[i - ch] if i >= ch else 0
            b = prev[i]
            c = prev[i - ch] if i >= ch else 0
            if f == 0:
                p = 0
            elif f == 1:
                p = a
            elif f == 2:
                p = b
            elif f == 3:
                p = (a + b) // 2
            else:
                pa, pb, pc = abs(b - c), abs(a - c), abs(a + b - 2 * c)
                p = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
            cur[i] = (line[i] + p) & 0xFF
        out[y] = cur
    out = out.astype(np.uint8)
    return out.reshape(h, w) if ch == 1 else out.reshape(h, w, 4)
