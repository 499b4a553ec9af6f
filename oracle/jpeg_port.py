"""numpy restatement of the baseline JPEG encoder of csrc/jpeg.cu: the CPU checker of its bytes.

It writes what `cv2.imencode('.jpg', bgr, [IMWRITE_JPEG_QUALITY, q])` writes with libjpeg-turbo's defaults, derived from ITU-T T.81
and checked against those files (tests/golden/reference_video_v1.npz):
  * JFIF 1.01 (density 1:1, no thumbnail), 4:2:0 sampling (Y 2x2, Cb / Cr 1x1), component ids 1 / 2 / 3, one interleaved scan,
    the Annex K.3 Huffman tables, no restart markers; markers SOI APP0 DQT(0) DQT(1) SOF0 DHT(DC0 AC0 DC1 AC1) SOS ... EOI;
  * quality q in [1, 100]: scale 5000 / q below 50, else 200 - 2 q; entry (K.1 / K.2 value * scale + 50) // 100 clamped to [1, 255];
  * colour conversion in 16-bit fixed point: Y = (19595 R + 38470 G + 7471 B + 2^15) >> 16,
    Cb = (-11059 R - 21709 G + 32768 B + (128 << 16) + 2^15 - 1) >> 16, Cr = (32768 R - 27439 G - 5329 B + (128 << 16) + 2^15 - 1) >> 16;
  * luma samples past the right / bottom edge repeat the last column / row up to whole 8 x 8 blocks; luma blocks wholly outside
    those (the rest of an edge MCU) are dummy blocks: zero AC, DC the quantised DC of the block before them in the MCU;
  * chroma: 2 x 2 sums of the edge-replicated full-resolution samples plus a bias 1, 2, 1, 2, ... along each row, >> 2; chroma rows
    past ceil(h / 2) repeat the last one;
  * the 8 x 8 integer FDCT of T.81 A.3.3 in the Loeffler-Ligtenberg-Moschytz factorisation with 13-bit constants and 2 extra bits
    between the passes (output scaled by 8), on samples - 128;
  * quantisation by 8 Q rounding half away from zero: sign(c) ((|c| + 4 Q) // (8 Q)).
"""
import numpy as np

ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

# T.81 Table K.1 / K.2, natural (row-major) order
LUMA_Q = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100,
    103, 99])
CHROMA_Q = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99]
    + [99] * 32)

# T.81 Table K.3-K.6: (BITS[1..16], HUFFVAL)
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
    0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
    0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa])


def huff_codes(table):
    """symbol -> (code, length) by T.81 Annex C (Figures C.1-C.3)"""
    bits, vals = table
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


def quant_tables(quality):
    """(luma, chroma) quantisation tables int64 [64], natural order"""
    if not 1 <= int(quality) <= 100:
        raise ValueError(f'quality must be in [1, 100], got {quality}')
    q = int(quality)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return tuple(np.clip((t * scale + 50) // 100, 1, 255).astype(np.int64) for t in (LUMA_Q, CHROMA_Q))


def header(h, w, quality):
    """every byte before the entropy-coded data"""
    out = bytearray(b'\xff\xd8')
    out += b'\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00'
    for tq, t in enumerate(quant_tables(quality)):
        out += bytes([0xff, 0xdb, 0, 67, tq]) + bytes(t[ZIGZAG].astype(np.uint8))
    out += bytes([0xff, 0xc0, 0, 17, 8, h >> 8, h & 255, w >> 8, w & 255, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1])
    for tc_th, (bits, vals) in ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA)):
        out += bytes([0xff, 0xc4, 0, 19 + len(vals), tc_th]) + bytes(bits) + bytes(vals)
    out += bytes([0xff, 0xda, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])
    return bytes(out)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, axis, first):
    """one pass of the integer FDCT along `axis` (int64 arrays); the first pass keeps 2 extra bits, the second removes them"""
    d = np.moveaxis(d, axis, -1)
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    sh = 11 if first else 15                                        # CONST_BITS - PASS1_BITS, CONST_BITS + PASS1_BITS
    o = [None] * 8
    if first:
        o[0], o[4] = (t10 + t11) << 2, (t10 - t11) << 2
    else:
        o[0], o[4] = _descale(t10 + t11, 2), _descale(t10 - t11, 2)
    z1 = (t12 + t13) * 4433
    o[2] = _descale(z1 + t13 * 6270, sh)
    o[6] = _descale(z1 - t12 * 15137, sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * 9633
    t4, t5, t6, t7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
    o[7] = _descale(t4 + z1 + z3, sh)
    o[5] = _descale(t5 + z2 + z4, sh)
    o[3] = _descale(t6 + z2 + z3, sh)
    o[1] = _descale(t7 + z1 + z4, sh)
    return np.moveaxis(np.stack(o, -1), -1, axis)


def fdct_quant(blocks, qt):
    """blocks int [..., 8, 8] of samples 0..255 -> quantised coefficients int64 [..., 64] in zigzag order"""
    d = blocks.astype(np.int64) - 128
    c = _fdct_1d(_fdct_1d(d, -1, True), -2, False).reshape(blocks.shape[:-2] + (64,))
    div = (qt * 8)[None]
    q = (np.abs(c) + (div >> 1)) // div
    return (np.sign(c) * q)[..., ZIGZAG]


def ycbcr(rgb):
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16
    return y, cb, cr


def mcu_coefficients(rgb, quality):
    """quantised coefficients int64 [mcu rows, mcu cols, 6, 64] (Y0 Y1 Y2 Y3 Cb Cr, zigzag) of an RGB u8 image [h, w, 3]"""
    h, w = rgb.shape[:2]
    my, mx = -(-h // 16), -(-w // 16)
    qy, qc = quant_tables(quality)
    y, cb, cr = ycbcr(rgb)
    rows, cols = np.minimum(np.arange(16 * my), h - 1), np.minimum(np.arange(16 * mx), w - 1)
    ypad = y[rows][:, cols]
    yb = ypad.reshape(my, 2, 8, mx, 2, 8).transpose(0, 3, 1, 4, 2, 5).reshape(my, mx, 4, 8, 8)
    ycoef = fdct_quant(yb, qy)
    # dummy luma blocks: block columns >= ceil(w / 8), block rows >= ceil(h / 8)
    bw, bh = -(-w // 8), -(-h // 8)
    for j in range(my):
        for i in range(mx):
            for k in range(4):
                if 2 * i + (k & 1) >= bw or 2 * j + (k >> 1) >= bh:
                    ycoef[j, i, k] = 0
                    ycoef[j, i, k, 0] = ycoef[j, i, k - 1, 0]
    ch = -(-h // 2)
    out = [ycoef]
    for c in (cb, cr):
        cpad = c[rows][:, cols].reshape(8 * my, 2, 8 * mx, 2).sum(axis=(1, 3))
        bias = np.where(np.arange(8 * mx) % 2 == 0, 1, 2)
        ds = (cpad + bias[None]) >> 2
        ds = ds[np.minimum(np.arange(8 * my), ch - 1)]
        cblk = ds.reshape(my, 8, mx, 8).transpose(0, 2, 1, 3)
        out.append(fdct_quant(cblk, qc)[:, :, None])
    return np.concatenate(out, axis=2)


class _Bits:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def put(self, code, length):
        self.acc = (self.acc << length) | code
        self.n += length
        while self.n >= 8:
            byte = (self.acc >> (self.n - 8)) & 255
            self.out.append(byte)
            if byte == 0xff:
                self.out.append(0)
            self.n -= 8
        self.acc &= (1 << self.n) - 1

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)
        return bytes(self.out)


def _category(v):
    return int(abs(int(v))).bit_length()


def entropy_code(coef):
    """the entropy-coded segment (stuffed, 1-padded) of coefficients [mcu rows, mcu cols, 6, 64]"""
    tabs = [(huff_codes(DC_LUMA), huff_codes(AC_LUMA)), (huff_codes(DC_CHROMA), huff_codes(AC_CHROMA))]
    bits = _Bits()
    pred = [0, 0, 0]
    flat = coef.reshape(-1, 6, 64)
    for mcu in flat:
        for b in range(6):
            comp = 0 if b < 4 else b - 3
            dc_t, ac_t = tabs[min(comp, 1)]
            blk = mcu[b]
            diff = int(blk[0]) - pred[comp]
            pred[comp] = int(blk[0])
            s = _category(diff)
            bits.put(*dc_t[s])
            if s:
                bits.put(diff & ((1 << s) - 1) if diff >= 0 else (diff - 1) & ((1 << s) - 1), s)
            run = 0
            for k in range(1, 64):
                v = int(blk[k])
                if v == 0:
                    run += 1
                    continue
                while run > 15:
                    bits.put(*ac_t[0xf0])
                    run -= 16
                s = _category(v)
                bits.put(*ac_t[(run << 4) | s])
                bits.put(v & ((1 << s) - 1) if v >= 0 else (v - 1) & ((1 << s) - 1), s)
                run = 0
            if run:
                bits.put(*ac_t[0x00])
    return bits.flush()


def encode(rgb, quality=95):
    """JFIF bytes of an RGB u8 image [h, w, 3], as cv2.imencode('.jpg', rgb[..., ::-1], [IMWRITE_JPEG_QUALITY, quality]) writes"""
    rgb = np.asarray(rgb)
    if rgb.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3 or min(rgb.shape[:2]) < 1 or max(rgb.shape[:2]) > 65535:
        raise ValueError(f'encode: RGB uint8 [h, w, 3] with 1 <= h, w <= 65535 expected, got {rgb.dtype} {rgb.shape}')
    h, w = rgb.shape[:2]
    return header(h, w, quality) + entropy_code(mcu_coefficients(rgb, quality)) + b'\xff\xd9'


def round_u8(x):
    """the fp32 prologue of the float encoder: rint(x * 255) in float32 (half to even), clamped to [0, 255]"""
    x = np.asarray(x, np.float32)
    return np.clip(np.rint(x * np.float32(255)), 0, 255).astype(np.uint8)
