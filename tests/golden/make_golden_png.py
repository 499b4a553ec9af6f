"""Pins for the PNG decoder (csrc/png_decode.cu): a corpus of PNG files written by OpenCV, PIL and a zlib-based writer here, with
the arrays `cv2.imread(path, cv2.IMREAD_COLOR)` returns for them (BGR -> RGB, uint8), and a malformed set derived from valid files,
each with the status the decoder must give (>= 0: a SSDNERF_PNG_* status; -1: the host chunk parser raises ValueError with `match`
in its message).

    python tests/golden/make_golden_png.py          (needs cv2 and PIL)
-> tests/golden/reference_png_v1.npz, replayed by tests/test_datasets_cpu.py and tests/test_png_decode_gpu.py.
"""
import io
import os
import struct
import tempfile
import zlib

import cv2
import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
SIG = b'\x89PNG\r\n\x1a\n'


def render_like(rng, h, w):
    """an RGBA object render: a shaded ellipse on a white, transparent background"""
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    cy, cx = h * rng.uniform(0.4, 0.6), w * rng.uniform(0.4, 0.6)
    ry, rx = h * rng.uniform(0.2, 0.35) + 0.5, w * rng.uniform(0.2, 0.35) + 0.5
    d = ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2
    inside = d < 1
    base = rng.uniform(0, 255, 3)
    shade = (1 - 0.6 * d)[..., None] * base + 20 * np.sin(x / 3 + y / 5)[..., None]
    rgb = np.where(inside[..., None], shade, 255.0)
    rgb = np.clip(rgb + rng.normal(0, 1.5, rgb.shape) * inside[..., None], 0, 255).astype(np.uint8)
    alpha = np.where(inside, 255, 0).astype(np.uint8)
    return np.concatenate([rgb, alpha[..., None]], -1)


def chunk(t, body):
    return struct.pack('>I', len(body)) + t + body + struct.pack('>I', zlib.crc32(t + body))


def ihdr(w, h, ct, depth=8, interlace=0):
    return chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, depth, ct, 0, 0, interlace))


def filter_rows(raw, bpp, filters):
    """raw uint8 [h, w * bpp] -> filtered stream with row r filtered by filters[r % len(filters)]"""
    h, n = raw.shape
    out = bytearray()
    prev = np.zeros(n, np.int32)
    for r in range(h):
        f = filters[r % len(filters)]
        cur = raw[r].astype(np.int32)
        left = np.concatenate([np.zeros(bpp, np.int32), cur[:-bpp]])
        ul = np.concatenate([np.zeros(bpp, np.int32), prev[:-bpp]])
        if f == 0:
            y = cur
        elif f == 1:
            y = cur - left
        elif f == 2:
            y = cur - prev
        elif f == 3:
            y = cur - (left + prev) // 2
        else:
            p = left + prev - ul
            pa, pb, pc = abs(p - left), abs(p - prev), abs(p - ul)
            y = cur - np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, prev, ul))
        out.append(f)
        out += (y & 255).astype(np.uint8).tobytes()
        prev = cur
    return bytes(out)


def write_png(raw, ct, filters=(0,), level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15, mem_level=8, idat_size=None, plte=None,
              extra=b''):
    h = raw.shape[0]
    bpp = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ct]
    w = raw.shape[1] // bpp
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, mem_level, strategy)
    z = c.compress(filter_rows(raw, bpp, filters)) + c.flush()
    return assemble(w, h, ct, z, idat_size, plte, extra)


def assemble(w, h, ct, z, idat_size=None, plte=None, extra=b''):
    out = SIG + ihdr(w, h, ct) + extra
    if plte is not None:
        out += chunk(b'PLTE', plte)
    step = idat_size or max(len(z), 1)
    for i in range(0, max(len(z), 1), step):
        out += chunk(b'IDAT', z[i:i + step])
    return out + chunk(b'IEND', b'')


def cv2_write(img, params):
    ok, buf = cv2.imencode('.png', img, params)
    assert ok
    return buf.tobytes()


def pil_write(im, **kw):
    b = io.BytesIO()
    im.save(b, format='PNG', **kw)
    return b.getvalue()


def valid_corpus(rng):
    files = []
    rgba = render_like(rng, 128, 128)
    bgra = rgba[..., [2, 1, 0, 3]]
    # OpenCV: colour types 6 / 2 / 0, levels 0-9, the five strategies
    for lvl in range(10):
        files.append((f'cv2_rgba_level{lvl}', cv2_write(bgra, [cv2.IMWRITE_PNG_COMPRESSION, lvl])))
    for st in range(5):
        files.append((f'cv2_rgba_strategy{st}', cv2_write(bgra, [cv2.IMWRITE_PNG_STRATEGY, st])))
    files.append(('cv2_rgb_default', cv2_write(bgra[..., :3].copy(), [])))
    files.append(('cv2_grey_default', cv2_write(cv2.cvtColor(bgra[..., :3], cv2.COLOR_BGR2GRAY), [])))
    # PIL: palette, grey + alpha, optimize=True
    im = Image.fromarray(rgba)
    files.append(('pil_rgba_optimize', pil_write(im, optimize=True)))
    files.append(('pil_palette', pil_write(im.convert('RGB').quantize(200))))
    files.append(('pil_palette_optimize', pil_write(im.convert('RGB').quantize(100), optimize=True)))
    pal_t = im.convert('RGB').quantize(32)
    pal_t.info['transparency'] = 0
    files.append(('pil_palette_trns', pil_write(pal_t, transparency=0)))
    files.append(('pil_la', pil_write(im.convert('LA'))))
    files.append(('pil_la_optimize', pil_write(im.convert('LA'), optimize=True)))
    # the writer here: every filter type alone and mixed per row, zlib strategies, windows, many blocks, many IDAT chunks
    raw6 = rgba.reshape(128, -1)
    for f in range(5):
        files.append((f'zlib_filter{f}', write_png(raw6, 6, filters=(f,))))
    files.append(('zlib_filters_mixed', write_png(raw6, 6, filters=(0, 1, 2, 3, 4, 4, 3, 1))))
    files.append(('zlib_filters_mixed_rgb', write_png(rgba[..., :3].reshape(128, -1), 2, filters=(4, 3, 2, 1, 0))))
    for name, st in (('filtered', zlib.Z_FILTERED), ('huffman', zlib.Z_HUFFMAN_ONLY), ('rle', zlib.Z_RLE), ('fixed', zlib.Z_FIXED)):
        files.append((f'zlib_{name}', write_png(raw6, 6, filters=(1, 4), level=9, strategy=st)))
    files.append(('zlib_window512', write_png(raw6, 6, filters=(4,), wbits=9)))
    files.append(('zlib_small_blocks', write_png(raw6, 6, filters=(2, 4), level=9, mem_level=1)))
    files.append(('zlib_level0_stored', write_png(raw6, 6, filters=(0,), level=0)))
    files.append(('zlib_idat_split_97', write_png(raw6, 6, filters=(1, 4), idat_size=97)))
    files.append(('zlib_idat_split_1', write_png(render_like(rng, 9, 11).reshape(9, -1), 6, filters=(4, 1), idat_size=1)))
    files.append(('zlib_text_chunk', write_png(raw6, 6, filters=(4,), extra=chunk(b'tEXt', b'Software\x00test'))))
    pal = rng.integers(0, 256, (7, 3), dtype=np.uint8)
    idx = rng.integers(0, 9, (13, 21), dtype=np.uint8)       # indices 7 and 8 lie past the 7-entry palette
    files.append(('zlib_palette_short', write_png(idx, 3, filters=(0, 1, 2, 3, 4), plte=pal.tobytes())))
    # sizes: 1 x 1, odd widths
    for (h, w) in ((1, 1), (5, 7), (3, 33), (2, 65), (31, 1), (17, 127)):
        img = render_like(rng, h, w)
        files.append((f'cv2_rgba_{h}x{w}', cv2_write(img[..., [2, 1, 0, 3]], [])))
        files.append((f'zlib_grey_{h}x{w}', write_png(img[..., 0].copy(), 0, filters=(4, 3, 1))))
        files.append((f'zlib_la_{h}x{w}', write_png(img[..., [1, 3]].reshape(h, -1), 4, filters=(3, 4))))
    return files


class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, v, n):              # least-significant bit first (deflate header fields, extra bits)
        self.bits += [(v >> i) & 1 for i in range(n)]

    def code(self, c, n):             # Huffman codes, most-significant bit first
        self.bits += [(c >> (n - 1 - i)) & 1 for i in range(n)]

    def bytes(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(sum(b[i + j] << j for j in range(8)) for i in range(0, len(b), 8))


def with_stream(png, z):
    """the same file with its zlib stream replaced (CRCs valid)"""
    w, h, _, ct = struct.unpack('>IIBB', png[16:26])
    plte = None
    pos = 8
    while pos < len(png):
        ln, t = struct.unpack('>I4s', png[pos:pos + 8])
        if t == b'PLTE':
            plte = png[pos + 8:pos + 8 + ln]
        pos += 12 + ln
    return assemble(w, h, ct, z, plte=plte)


def zlib_stream(png):
    pos, z = 8, b''
    while pos < len(png):
        ln, t = struct.unpack('>I4s', png[pos:pos + 8])
        if t == b'IDAT':
            z += png[pos + 8:pos + 8 + ln]
        pos += 12 + ln
    return z


def fixed_block(ops):
    """zlib stream of one final fixed-Huffman block: ops are ('lit', byte) / ('sym', litlen symbol) / ('dist', symbol)"""
    bw = BitWriter()
    bw.put(1, 1)
    bw.put(1, 2)
    for kind, v in ops:
        if kind == 'dist':
            bw.code(v, 5)
        elif v < 144:
            bw.code(0x30 + v, 8)
        elif v < 256:
            bw.code(0x190 + v - 144, 9)
        elif v < 280:
            bw.code(v - 256, 7)
        else:
            bw.code(0xC0 + v - 280, 8)
    return b'\x78\x01' + bw.bytes()


def malformed_corpus(valid):
    good = dict(valid)
    base = good['cv2_rgba_5x7']
    z = zlib_stream(base)
    out = []
    for cut in (1, 2, 7, len(z) // 2, len(z) - 4, len(z) - 1):
        out.append((f'stream_truncated_{cut}', with_stream(base, z[:cut]), 1, ''))
    out.append(('zlib_cm_flipped', with_stream(base, bytes([z[0] ^ 0x01]) + z[1:]), 2, ''))
    out.append(('zlib_fcheck_flipped', with_stream(base, z[:1] + bytes([z[1] ^ 0x01]) + z[2:]), 2, ''))
    fd = bytes([0x78, 0x20 | (31 - (0x7820 % 31))])
    out.append(('zlib_fdict_set', with_stream(base, fd + z[2:]), 2, ''))
    out.append(('zlib_window_64k', with_stream(base, bytes([0x88, 31 - (0x8800 % 31)]) + z[2:]), 2, ''))
    out.append(('block_type_3', with_stream(base, b'\x78\x01\x07\x00'), 3, ''))
    stored = zlib_stream(good['zlib_level0_stored'])
    out.append(('stored_nlen_flipped', with_stream(good['zlib_level0_stored'], stored[:5] + bytes([stored[5] ^ 0x10]) + stored[6:]), 4, ''))
    bw = BitWriter()                  # dynamic block whose code-length code gives four symbols one bit each
    bw.put(1, 1); bw.put(2, 2); bw.put(0, 5); bw.put(0, 5); bw.put(0, 4)
    for _ in range(4):
        bw.put(1, 3)
    out.append(('code_lengths_oversubscribed', with_stream(base, b'\x78\x01' + bw.bytes() + b'\x00' * 8), 5, ''))
    bw = BitWriter()                  # ... and one whose code-length code is incomplete (a single 2-bit code)
    bw.put(1, 1); bw.put(2, 2); bw.put(0, 5); bw.put(0, 5); bw.put(0, 4)
    bw.put(2, 3); bw.put(0, 3); bw.put(0, 3); bw.put(0, 3)
    out.append(('code_lengths_incomplete', with_stream(base, b'\x78\x01' + bw.bytes() + b'\x00' * 8), 5, ''))
    out.append(('distance_before_start', with_stream(base, fixed_block([('sym', 0), ('sym', 257), ('dist', 1), ('sym', 256)]) + b'\0' * 4), 7, ''))
    out.append(('litlen_symbol_286', with_stream(base, fixed_block([('sym', 0), ('sym', 286)]) + b'\0' * 4), 6, ''))
    out.append(('dist_symbol_30', with_stream(base, fixed_block([('sym', 0), ('sym', 0), ('sym', 257), ('dist', 30)]) + b'\0' * 4), 6, ''))
    out.append(('adler_flipped', with_stream(base, z[:-1] + bytes([z[-1] ^ 0x01])), 11, ''))
    raw = np.full((5, 7 * 4), 9, np.uint8)
    filt = bytearray(filter_rows(raw, 4, (0,)))
    filt[2 * 29] = 5
    out.append(('filter_byte_5', with_stream(base, zlib.compress(bytes(filt))), 10, ''))
    out.append(('too_much_data', with_stream(base, zlib.compress(bytes(filt) + b'\0')), 8, ''))
    out.append(('too_little_data', with_stream(base, zlib.compress(bytes(filt[:-1]))), 9, ''))
    # host-side refusals
    bad_crc = bytearray(base)
    bad_crc[8 + 8 + 13] ^= 1
    out.append(('bad_ihdr_crc', bytes(bad_crc), -1, 'bad CRC'))
    idat_at = base.index(b'IDAT')
    bad_crc = bytearray(base)
    bad_crc[idat_at + 6] ^= 1
    out.append(('bad_idat_crc', bytes(bad_crc), -1, 'bad CRC'))
    out.append(('missing_iend', base[:-12], -1, 'IEND'))
    out.append(('file_truncated', base[:len(base) // 2], -1, 'past the end'))
    out.append(('bad_signature', b'\x89PNG\r\n\x1a\x00' + base[8:], -1, 'signature'))
    huge = SIG + chunk(b'IHDR', struct.pack('>IIBBBBB', 100000, 100000, 8, 6, 0, 0, 0)) + base[33:]
    out.append(('absurd_ihdr_size', huge, -1, 'can hold'))
    return out


def main():
    rng = np.random.default_rng(20261017)
    valid = valid_corpus(rng)
    arrays = []
    with tempfile.TemporaryDirectory() as d:
        for name, data in valid:
            p = os.path.join(d, name + '.png')
            with open(p, 'wb') as f:
                f.write(data)
            img = cv2.imread(p, cv2.IMREAD_COLOR)
            assert img is not None, name
            arrays.append(np.ascontiguousarray(img[..., ::-1]))
    mal = malformed_corpus(valid)

    def pack(blobs):
        offs = np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64)
        return np.frombuffer(b''.join(blobs), np.uint8), offs
    vb, vo = pack([d for _, d in valid])
    mb, mo = pack([d for _, d, _, _ in mal])
    np.savez_compressed(
        os.path.join(HERE, 'reference_png_v1.npz'),
        valid_names=np.array([n for n, _ in valid]), valid_bytes=vb, valid_offsets=vo,
        valid_shapes=np.array([a.shape for a in arrays], np.int64), valid_pixels=np.concatenate([a.ravel() for a in arrays]),
        mal_names=np.array([n for n, *_ in mal]), mal_bytes=mb, mal_offsets=mo,
        mal_status=np.array([s for *_, s, _ in mal], np.int32), mal_match=np.array([m for *_, m in mal]),
        cv2_version=np.array(cv2.__version__))
    print(len(valid), 'valid files,', len(mal), 'malformed;', os.path.getsize(os.path.join(HERE, 'reference_png_v1.npz')), 'bytes')


if __name__ == '__main__':
    main()
