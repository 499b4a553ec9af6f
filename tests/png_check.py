"""A stdlib + numpy PNG reader for the viz tests: chunk CRCs checked with zlib.crc32, the zlib stream inflated with zlib.decompress
(which checks Adler-32), all five filter types undone in numpy.  It reads exactly what csrc/png.cu writes: 8-bit RGBA, non-interlaced."""
import struct
import zlib

import numpy as np

SIGNATURE = b'\x89PNG\r\n\x1a\n'


def chunks(data):
    """[(type, body)] after checking the signature and every chunk's CRC"""
    assert data[:8] == SIGNATURE, 'bad signature'
    out, pos = [], 8
    while pos < len(data):
        (n,) = struct.unpack('>I', data[pos:pos + 4])
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        (crc,) = struct.unpack('>I', data[pos + 8 + n:pos + 12 + n])
        assert zlib.crc32(kind + body) == crc, f'bad CRC in {kind}'
        out.append((kind, body))
        pos += 12 + n
    assert pos == len(data) and out[-1] == (b'IEND', b''), 'bad chunk layout'
    return out


def unfilter(raw, h, w):
    """uint8 [h, w, 4] from the filtered stream (filter byte + 4 w bytes per row)"""
    rows = np.frombuffer(raw, np.uint8).reshape(h, 4 * w + 1)
    out = np.zeros((h, 4 * w), np.int32)
    prev = np.zeros(4 * w, np.int32)
    for y in range(h):
        t, f = rows[y, 0], rows[y, 1:].astype(np.int32)
        if t == 0:
            cur = f
        elif t == 1:
            cur = np.cumsum(f.reshape(w, 4), axis=0).reshape(-1) % 256
        elif t == 2:
            cur = (f + prev) % 256
        elif t in (3, 4):
            cur = np.zeros(4 * w, np.int32)
            a = np.zeros(4, np.int32)
            c = np.zeros(4, np.int32)
            for x in range(w):
                b = prev[4 * x:4 * x + 4]
                if t == 3:
                    pr = (a + b) // 2
                else:
                    p = a + b - c
                    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
                    pr = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
                a = (f[4 * x:4 * x + 4] + pr) % 256
                cur[4 * x:4 * x + 4] = a
                c = b
        else:
            raise AssertionError(f'bad filter type {t} in row {y}')
        out[y] = cur
        prev = cur
    return out.astype(np.uint8).reshape(h, w, 4)


def decode(data):
    """(pixels uint8 [h, w, 4], filtered stream bytes, deflate payload bytes) of an 8-bit RGBA PNG"""
    cs = chunks(data)
    assert cs[0][0] == b'IHDR'
    w, h, depth, ctype, comp, filt, interlace = struct.unpack('>IIBBBBB', cs[0][1])
    assert (depth, ctype, comp, filt, interlace) == (8, 6, 0, 0, 0)
    idat = b''.join(body for kind, body in cs if kind == b'IDAT')
    raw = zlib.decompress(idat)
    assert len(raw) == h * (4 * w + 1)
    return unfilter(raw, h, w), raw, len(idat) - 6
