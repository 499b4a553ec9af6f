"""numpy statement of the H.264 all-intra encoder of csrc/h264.cu (C ABI section 13), and of the decoder-side deblocking filter that
turns its reconstruction into the picture a decoder outputs.

The bitstream subset (ITU-T H.264 clause numbers in brackets):
  * Constrained Baseline (profile_idc 66, constraint_set0 and constraint_set1), 8-bit 4:2:0, CAVLC, progressive frames.  SPS: the
    smallest Table A-1 level whose MaxFS, MaxMBPS and frame-dimension limits fit (MaxBR, MaxCPB are not checked; a rate above level
    5.2's MaxMBPS is signalled as 5.2), pic_order_cnt_type 2, max_num_ref_frames 0, cropping to the frame size, VUI with square
    pixels, limited range, colour primaries / transfer / matrix 6 (BT.601, SMPTE 170M) and max_num_reorder_frames 0.  PPS:
    pic_init_qp = QP, chroma_qp_index_offset 0, deblocking with the default controls (enabled, offsets 0).
  * Every frame is one IDR access unit of one I slice (frame_num 0, idr_pic_id alternating 0 / 1 with the frame index, slice_qp_delta
    0) and alternating over a video's frames; every macroblock is I_16x16 with mb_qp_delta 0.
  * Mode decision: luma V (0), H (1), DC (2), Plane (3) and chroma DC (0), H (1), V (2), Plane (3) among those whose neighbours
    exist; the mode of least SATD (sum over the 4x4 blocks of |4x4 Hadamard of the residual|, Cb + Cr for chroma); ties to the
    lowest mode number.
  * Forward quantisation (MF of the standard's derivation, intra offset f = 2^qbits / 3, qbits = 15 + QP / 6):
      AC:            |l| = (|w| MF(QP % 6, pos) + f) >> qbits
      Intra16x16 DC: |l| = (|y| MF(QP % 6, 0) + 4 f) >> (qbits + 2), y the unscaled 4x4 Hadamard of the 16 DC terms (the standard's
                     (|y / 2| MF + 2 f) >> (qbits + 1) without truncating y / 2)
      chroma DC:     |l| = (|y| MF(QP % 6, 0) + 2 f) >> (qbits + 1), y the 2x2 Hadamard of the 4 DC terms
    sign(l) = sign(w).  Chroma uses QPc of Table 8-15.  Dequantisation, the DC inverse transforms and the 4x4 inverse transform are
    clause 8.5's, so the reconstruction is the decoder's picture before deblocking.
  * QP range: MIN_QP .. 51.  Baseline caps level_prefix at 15, which codes |level| <= 2063 at any suffixLength (suffixLength 0 or 1:
    levelCode <= 30 + 4095 = 4125 -> |level| <= 2063; larger suffixLengths reach further).  For 8-bit input |residual| <= 255, so
    |w| <= 255 (sum |row u|)(sum |row v|) of the core transform rows (4, 6, 4, 6): 9180 at odd/odd, 6120 at mixed, 4080 at even/even
    positions; a DC term is at most 16 x 255 = 4080, the 4x4 Hadamard of 16 of them at most 65280 (quantised with the extra shift),
    the 2x2 one of 4 at most 16320.
    level_bound(qp) evaluates these through the quantiser; MIN_QP is the smallest QP from which every bound is <= 2063 (I_PCM, which
    would lift the limit, is not used: its byte alignment would make a macroblock's bit length depend on where it starts).
  * Colour: 8-bit BT.601 limited range, Y = ((66 R + 129 G + 25 B + 128) >> 8) + 16, Cb = ((-38 R - 74 G + 112 B + 128) >> 8) + 128,
    Cr = ((112 R - 94 G - 18 B + 128) >> 8) + 128 per pixel (arithmetic shifts); chroma planes the rounded 2x2 mean
    (a + b + c + d + 2) >> 2.  Even sizes only; the planes are padded to whole macroblocks by edge replication (luma to 16, chroma to
    8) and the SPS crops the padding.
"""
import numpy as np

MAX_LEVEL = 2063
MAX_FS = 36864                        # level 5.2
MAX_DIM_MBS = 543                     # floor(sqrt(8 MaxFS)) of level 5.2

# ------------------------------------------------------------------------------------------------ tables
LEVELS = [  # (level_idc, MaxMBPS, MaxFS) of Table A-1 (level 1b is skipped)
    (10, 1485, 99), (11, 3000, 396), (12, 6000, 396), (13, 11880, 396), (20, 11880, 396), (21, 19800, 792), (22, 20250, 1620),
    (30, 40500, 1620), (31, 108000, 3600), (32, 216000, 5120), (40, 245760, 8192), (41, 245760, 8192), (42, 522240, 8704),
    (50, 589824, 22080), (51, 983040, 36864), (52, 2073600, 36864)]

MF = np.array([[13107, 5243, 8066], [11916, 4660, 7490], [10082, 4194, 6554], [9362, 3647, 5825], [8192, 3355, 5243],
               [7282, 2893, 4559]], np.int64)
V = np.array([[10, 16, 13], [11, 18, 14], [13, 20, 16], [14, 23, 18], [16, 25, 20], [18, 29, 23]], np.int64)
POS = np.array([[0, 2, 0, 2], [2, 1, 2, 1], [0, 2, 0, 2], [2, 1, 2, 1]])        # 0 even/even, 1 odd/odd, 2 mixed
ZIGZAG = np.array([0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15])       # scan index -> raster index of a 4x4 block
QPC = list(range(30)) + [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39]
CF = np.array([[1, 1, 1, 1], [2, 1, -1, -2], [1, -1, -1, 1], [1, -2, 2, -1]], np.int64)
H4 = np.array([[1, 1, 1, 1], [1, 1, -1, -1], [1, -1, -1, 1], [1, -1, 1, -1]], np.int64)
H2 = np.array([[1, 1], [1, -1]], np.int64)

# Table 9-5 coeff_token as (length, code), index 4 TotalCoeff + TrailingOnes; columns 0 <= nC < 2, 2 <= nC < 4, 4 <= nC < 8, 8 <= nC
CT_LEN = [
    [1, 0, 0, 0, 6, 2, 0, 0, 8, 6, 3, 0, 9, 8, 7, 5, 10, 9, 8, 6, 11, 10, 9, 7, 13, 11, 10, 8, 13, 13, 11, 9, 13, 13, 13, 10,
     14, 14, 13, 11, 14, 14, 14, 13, 15, 15, 14, 14, 15, 15, 15, 14, 16, 15, 15, 15, 16, 16, 16, 15, 16, 16, 16, 16, 16, 16, 16, 16],
    [2, 0, 0, 0, 6, 2, 0, 0, 6, 5, 3, 0, 7, 6, 6, 4, 8, 6, 6, 4, 8, 7, 7, 5, 9, 8, 8, 6, 11, 9, 9, 6, 11, 11, 11, 7,
     12, 11, 11, 9, 12, 12, 12, 11, 12, 12, 12, 11, 13, 13, 13, 12, 13, 13, 13, 13, 13, 14, 13, 13, 14, 14, 14, 13, 14, 14, 14, 14],
    [4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4, 7, 5, 5, 4, 7, 5, 5, 4, 7, 6, 6, 4, 7, 6, 6, 4, 8, 7, 7, 5,
     8, 8, 7, 6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10],
    [6 if i == 0 or (i >= 4 and (i & 3) <= min(i >> 2, 3)) else 0 for i in range(68)]]
CT_CODE = [
    [1, 0, 0, 0, 5, 1, 0, 0, 7, 4, 1, 0, 7, 6, 5, 3, 7, 6, 5, 3, 7, 6, 5, 4, 15, 6, 5, 4, 11, 14, 5, 4, 8, 10, 13, 4,
     15, 14, 9, 4, 11, 10, 13, 12, 15, 14, 9, 12, 11, 10, 13, 8, 15, 1, 9, 12, 11, 14, 13, 8, 7, 10, 9, 12, 4, 6, 5, 8],
    [3, 0, 0, 0, 11, 2, 0, 0, 7, 7, 3, 0, 7, 10, 9, 5, 7, 6, 5, 4, 4, 6, 5, 6, 7, 6, 5, 8, 15, 6, 5, 4, 11, 14, 13, 4,
     15, 10, 9, 4, 11, 14, 13, 12, 8, 10, 9, 8, 15, 14, 13, 12, 11, 10, 9, 12, 7, 11, 6, 8, 9, 8, 10, 1, 7, 6, 5, 4],
    [15, 0, 0, 0, 15, 14, 0, 0, 11, 15, 13, 0, 8, 12, 14, 12, 15, 10, 11, 11, 11, 8, 9, 10, 9, 14, 13, 9, 8, 10, 9, 8, 15, 14, 13, 13,
     11, 14, 10, 12, 15, 10, 13, 12, 11, 14, 9, 12, 8, 10, 13, 8, 13, 7, 9, 12, 9, 12, 11, 10, 5, 8, 7, 6, 1, 4, 3, 2],
    [3, 0, 0, 0] + [i - 4 for i in range(4, 68)]]      # 8 <= nC: 6-bit (TotalCoeff - 1, TrailingOnes), TotalCoeff 0 is 000011
CT_DC_LEN = [2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7]         # nC == -1 (chroma DC)
CT_DC_CODE = [1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0]
# Tables 9-7 / 9-8 total_zeros of 4x4 blocks, row TotalCoeff - 1, column total_zeros; 9-9a of chroma DC
TZ_LEN = [[1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9], [3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6],
          [4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6], [5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5], [4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5],
          [6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6], [6, 5, 3, 3, 3, 2, 3, 4, 3, 6], [6, 4, 5, 3, 2, 2, 3, 3, 6], [6, 6, 4, 2, 2, 3, 2, 5],
          [5, 5, 3, 2, 2, 2, 4], [4, 4, 3, 3, 1, 3], [4, 4, 2, 1, 3], [3, 3, 1, 2], [2, 2, 1], [1, 1]]
TZ_CODE = [[1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1], [7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0],
           [5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0], [3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0], [5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0],
           [1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 5, 4, 3, 3, 2, 1, 1, 0], [1, 1, 1, 3, 3, 2, 2, 1, 0], [1, 0, 1, 3, 2, 1, 1, 1],
           [1, 0, 1, 3, 2, 1, 1], [0, 1, 1, 2, 1, 3], [0, 1, 1, 1, 1], [0, 1, 1, 1], [0, 1, 1], [0, 1]]
TZ_DC_LEN = [[1, 2, 3, 3], [1, 2, 2], [1, 1]]
TZ_DC_CODE = [[1, 1, 1, 0], [1, 1, 0], [1, 0]]
# Table 9-10 run_before, row min(zerosLeft, 7) - 1, column run_before
RB_LEN = [[1, 1], [1, 2, 2], [2, 2, 2, 2], [2, 2, 2, 3, 3], [2, 2, 3, 3, 3, 3], [2, 3, 3, 3, 3, 3, 3],
          [3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11]]
RB_CODE = [[1, 0], [1, 1, 0], [3, 2, 1, 0], [3, 2, 1, 1, 0], [3, 2, 3, 2, 1, 0], [3, 0, 1, 3, 2, 5, 4],
           [7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1]]
# Tables 8-16 / 8-17: alpha', beta' and tC0 at bS 3 by indexA / indexB
ALPHA = [0] * 16 + [4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25, 28, 32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113, 127,
                    144, 162, 182, 203, 226, 255, 255]
BETA = [0] * 16 + [2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16, 17,
                   17, 18, 18]
TC0_BS3 = [0] * 17 + [1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 4, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 23, 25]


def level_bound(qp):
    """the largest |level| 8-bit input can produce at `qp` (AC, Intra16x16 DC and chroma DC paths; see the module docstring)"""
    def ac(q):
        qb, fo = 15 + q // 6, (1 << (15 + q // 6)) // 3
        return max((w * MF[q % 6, p] + fo) >> qb for w, p in ((4080, 0), (9180, 1), (6120, 2)))

    def dc(q, y, extra):
        qb, fo = 15 + q // 6, (1 << (15 + q // 6)) // 3
        return (y * MF[q % 6, 0] + (2 << extra) * fo) >> (qb + 1 + extra)
    qc = QPC[qp]
    return int(max(ac(qp), ac(qc), dc(qp, 65280, 1), dc(qc, 16320, 0)))


MIN_QP = next(q for q in range(52) if all(level_bound(r) <= MAX_LEVEL for r in range(q, 52)))


def level_idc(h, w, fps):
    """the smallest Table A-1 level whose MaxFS, frame-dimension and MaxMBPS limits hold (5.2 when no level's MaxMBPS does)"""
    from fractions import Fraction
    mw, mh = (w + 15) // 16, (h + 15) // 16
    fs = mw * mh
    fps = Fraction(fps)
    for idc, mbps, maxfs in LEVELS:
        if fs <= maxfs and mw * mw <= 8 * maxfs and mh * mh <= 8 * maxfs and fs * fps <= mbps:
            return idc
    return 52


def check_args(h, w, qp):
    if h < 2 or w < 2 or h % 2 or w % 2:
        raise ValueError(f'h264: even h, w >= 2 expected, got {h} x {w}')
    mw, mh = (w + 15) // 16, (h + 15) // 16
    if mw * mh > MAX_FS or mw > MAX_DIM_MBS or mh > MAX_DIM_MBS:
        raise ValueError(f'h264: {h} x {w} exceeds level 5.2 ({MAX_FS} macroblocks, {MAX_DIM_MBS} per side)')
    if not MIN_QP <= qp <= 51:
        raise ValueError(f'h264: qp must be in [{MIN_QP}, 51], got {qp}')


# ------------------------------------------------------------------------------------------------ bits
class Bits:
    def __init__(self):
        self.v, self.n = 0, 0

    def u(self, value, n):
        value, n = int(value), int(n)
        assert 0 <= value < (1 << n) or n == 0 and value == 0, (value, n)
        self.v = (self.v << n) | value
        self.n += n

    def ue(self, k):
        m = (k + 1).bit_length()
        self.u(0, m - 1)
        self.u(k + 1, m)

    def se(self, k):
        self.ue(2 * k - 1 if k > 0 else -2 * k)

    def extend(self, other):
        self.v = (self.v << other.n) | other.v
        self.n += other.n

    def trailing(self):
        """rbsp_trailing_bits: the stop bit and zero bits to the byte boundary"""
        self.u(1, 1)
        self.u(0, (8 - self.n % 8) % 8)

    def bytes(self):
        assert self.n % 8 == 0
        return self.v.to_bytes(self.n // 8, 'big')


def ep_bytes(rbsp):
    """emulation prevention: 0x03 after every two zero bytes that precede a byte <= 3 (7.4.1, sequentially)"""
    out, zeros = bytearray(), 0
    for b in rbsp:
        if zeros == 2 and b <= 3:
            out.append(3)
            zeros = 0
        out.append(b)
        zeros = zeros + 1 if b == 0 else 0
    return bytes(out)


def nal(nal_byte, rbsp):
    return bytes([nal_byte]) + ep_bytes(rbsp)


def residual_block(bs, coeffs, nc, max_coeff):
    """CAVLC residual_block (9.2) of `coeffs` (scan order, max_coeff of them) with nC `nc`; returns TotalCoeff"""
    nz = [i for i, c in enumerate(coeffs) if c]
    tc = len(nz)
    t1 = 0
    for i in reversed(nz):
        if abs(coeffs[i]) != 1 or t1 == 3:
            break
        t1 += 1
    idx = 4 * tc + t1
    if nc == -1:
        bs.u(CT_DC_CODE[idx], CT_DC_LEN[idx])
    else:
        col = 0 if nc < 2 else 1 if nc < 4 else 2 if nc < 8 else 3
        bs.u(CT_CODE[col][idx], CT_LEN[col][idx])
    if tc == 0:
        return 0
    levels = [coeffs[i] for i in reversed(nz)]
    for i in range(t1):
        bs.u(1 if levels[i] < 0 else 0, 1)
    sl = 1 if tc > 10 and t1 < 3 else 0
    for i in range(t1, tc):
        lv = levels[i]
        code = 2 * lv - 2 if lv > 0 else -2 * lv - 1
        if i == t1 and t1 < 3:
            code -= 2
        if sl == 0 and code < 14:
            bs.u(1, code + 1)
        elif sl == 0 and code < 30:
            bs.u(1, 15)
            bs.u(code - 14, 4)
        elif sl > 0 and code < (15 << sl):
            bs.u(1, (code >> sl) + 1)
            bs.u(code & ((1 << sl) - 1), sl)
        else:
            esc = code - (30 if sl == 0 else 15 << sl)
            assert esc < 4096, f'level {lv} does not fit level_prefix 15'
            bs.u(1, 16)
            bs.u(esc, 12)
        if sl == 0:
            sl = 1
        if abs(lv) > (3 << (sl - 1)) and sl < 6:
            sl += 1
    if tc < max_coeff:
        tz = nz[-1] + 1 - tc
        if max_coeff == 4:
            bs.u(TZ_DC_CODE[tc - 1][tz], TZ_DC_LEN[tc - 1][tz])
        else:
            bs.u(TZ_CODE[tc - 1][tz], TZ_LEN[tc - 1][tz])
    else:
        tz = 0
    left = tz
    for k in range(tc - 1):
        if left == 0:
            break
        run = nz[tc - 1 - k] - nz[tc - 2 - k] - 1
        r = min(left, 7) - 1
        bs.u(RB_CODE[r][run], RB_LEN[r][run])
        left -= run
    return tc


# ------------------------------------------------------------------------------------------------ colour
def round_u8(x):
    """the fp32 prologue: rint(x * 255) in float32, clamped to [0, 255] (NaN -> 0)"""
    v = np.rint(np.asarray(x, np.float32) * np.float32(255))
    return np.nan_to_num(np.clip(v, 0, 255), nan=0).astype(np.uint8)


def yuv420(rgb):
    """padded planes (Y [16 mh, 16 mw], Cb, Cr [8 mh, 8 mw]) int64 of an even-sized u8 RGB frame"""
    h, w, _ = rgb.shape
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    y = ((66 * r + 129 * g + 25 * b + 128) >> 8) + 16
    cb = ((-38 * r - 74 * g + 112 * b + 128) >> 8) + 128
    cr = ((112 * r - 94 * g - 18 * b + 128) >> 8) + 128
    sub = lambda c: (c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2] + 2) >> 2
    mh, mw = (h + 15) // 16, (w + 15) // 16
    pad = lambda p, s: np.pad(p, ((0, s * mh - p.shape[0]), (0, s * mw - p.shape[1])), mode='edge')
    return pad(y, 16), pad(sub(cb), 8), pad(sub(cr), 8)


# ------------------------------------------------------------------------------------------------ prediction
def pred_modes(rec, x0, y0, n, chroma):
    """{mode: n x n prediction} of the available intra 16x16 (n 16) or chroma (n 8) modes of the block at (x0, y0) of plane rec"""
    top = rec[y0 - 1, x0:x0 + n] if y0 > 0 else None
    left = rec[y0:y0 + n, x0 - 1] if x0 > 0 else None
    out = {}
    if chroma:
        dc = np.zeros((n, n), np.int64)
        for by in range(2):
            for bx in range(2):
                t = top[4 * bx:4 * bx + 4].sum() if top is not None else None
                l = left[4 * by:4 * by + 4].sum() if left is not None else None
                if (bx, by) in ((0, 0), (1, 1)):
                    v = (t + l + 4) >> 3 if t is not None and l is not None else (l + 2) >> 2 if l is not None else \
                        (t + 2) >> 2 if t is not None else 128
                elif by == 0:
                    v = (t + 2) >> 2 if t is not None else (l + 2) >> 2 if l is not None else 128
                else:
                    v = (l + 2) >> 2 if l is not None else (t + 2) >> 2 if t is not None else 128
                dc[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = v
        out[0] = dc
        if left is not None:
            out[1] = np.repeat(left[:, None], n, 1)
        if top is not None:
            out[2] = np.repeat(top[None, :], n, 0)
    else:
        if top is not None:
            out[0] = np.repeat(top[None, :], n, 0)
        if left is not None:
            out[1] = np.repeat(left[:, None], n, 1)
        if top is not None and left is not None:
            v = (top.sum() + left.sum() + 16) >> 5
        elif left is not None:
            v = (left.sum() + 8) >> 4
        elif top is not None:
            v = (top.sum() + 8) >> 4
        else:
            v = 128
        out[2] = np.full((n, n), v, np.int64)
    if top is not None and left is not None:
        corner = rec[y0 - 1, x0 - 1]
        t = np.concatenate([[corner], top])          # t[k + 1] = p[k, -1]
        l = np.concatenate([[corner], left])
        half = n // 2
        k = np.arange(1, half + 1)
        hh = int((k * (t[half + k] - t[half - k])).sum())
        vv = int((k * (l[half + k] - l[half - k])).sum())
        s = 5 if n == 16 else 34
        sh = 6
        b, c = (s * hh + 32) >> sh, (s * vv + 32) >> sh
        a = 16 * (int(left[-1]) + int(top[-1]))
        yy, xx = np.mgrid[0:n, 0:n]
        out[3] = np.clip((a + b * (xx - (half - 1)) + c * (yy - (half - 1)) + 16) >> 5, 0, 255)
    return out


def blocks4(p):
    """[n/4 rows, n/4 cols, 4, 4] view of an n x n array"""
    n = p.shape[0]
    return p.reshape(n // 4, 4, n // 4, 4).transpose(0, 2, 1, 3)


def satd(res):
    b = blocks4(res)
    return int(np.abs(H4 @ b @ H4).sum())


# ------------------------------------------------------------------------------------------------ transform and quantisation
def quant_ac(w, qp):
    qb, fo = 15 + qp // 6, (1 << (15 + qp // 6)) // 3
    mf = MF[qp % 6][POS]
    return np.sign(w) * ((np.abs(w) * mf + fo) >> qb)


def quant_dc(y, qp, chroma):
    """DC levels of the unscaled Hadamard y: the standard's luma path halves it first (here exactly, by one more shift)"""
    qb, fo = 15 + qp // 6, (1 << (15 + qp // 6)) // 3
    if chroma:
        return np.sign(y) * ((np.abs(y) * MF[qp % 6, 0] + 2 * fo) >> (qb + 1))
    return np.sign(y) * ((np.abs(y) * MF[qp % 6, 0] + 4 * fo) >> (qb + 2))


def dequant_ac(c, qp):
    ls = 16 * V[qp % 6][POS]
    if qp >= 24:
        return (c * ls) << (qp // 6 - 4)
    return (c * ls + (1 << (3 - qp // 6))) >> (4 - qp // 6)


def inv4(d):
    """8.5.12.2 on [..., 4, 4] (rows then columns), (h + 32) >> 6"""
    def one(x):     # along the last axis
        e0, e1 = x[..., 0] + x[..., 2], x[..., 0] - x[..., 2]
        e2, e3 = (x[..., 1] >> 1) - x[..., 3], x[..., 1] + (x[..., 3] >> 1)
        return np.stack([e0 + e3, e1 + e2, e1 - e2, e0 - e3], -1)
    f = one(d)
    g = one(np.swapaxes(f, -1, -2))
    return (np.swapaxes(g, -1, -2) + 32) >> 6


def code_plane(src, pred, qp, chroma):
    """levels and reconstruction of one 16x16 luma or 8x8 chroma block of I_16x16: (dc levels [k, k] of the block grid,
    ac levels [k, k, 16] raster with 0 at the DC, reconstruction)"""
    res = src - pred
    w = CF @ blocks4(res) @ CF.T                    # [k, k, 4, 4]
    k = w.shape[0]
    hm = H2 if chroma else H4
    dcl = quant_dc(hm @ w[:, :, 0, 0] @ hm, qp, chroma)
    acl = quant_ac(w, qp)
    acl[:, :, 0, 0] = 0
    # decoder side
    f = hm @ dcl @ hm
    ls0 = 16 * V[qp % 6, 0]
    if chroma:
        dcv = ((f * ls0) << (qp // 6)) >> 5
    elif qp >= 36:
        dcv = (f * ls0) << (qp // 6 - 6)
    else:
        dcv = (f * ls0 + (1 << (5 - qp // 6))) >> (6 - qp // 6)
    d = dequant_ac(acl, qp)
    d[:, :, 0, 0] = dcv
    r = inv4(d)
    rec = np.clip(pred + r.transpose(0, 2, 1, 3).reshape(4 * k, 4 * k), 0, 255)
    return dcl, acl.reshape(k, k, 16), rec


def encode_picture(rgb, qp, idr_pic_id=0):
    """(slice NAL unit bytes, reconstruction planes before deblocking (Y, Cb, Cr), padded) of one u8 RGB frame"""
    y, cb, cr = yuv420(rgb)
    H, W = y.shape
    mh, mw = H // 16, W // 16
    qpc = QPC[qp]
    ry, rcb, rcr = np.zeros_like(y), np.zeros_like(cb), np.zeros_like(cr)
    tcy = np.zeros((4 * mh, 4 * mw), np.int64)
    tcc = np.zeros((2, 2 * mh, 2 * mw), np.int64)

    def nc_of(tc, gy, gx):
        a, b = gx > 0, gy > 0
        if a and b:
            return (tc[gy, gx - 1] + tc[gy - 1, gx] + 1) >> 1
        return tc[gy, gx - 1] if a else tc[gy - 1, gx] if b else 0

    bs = Bits()
    bs.ue(0)                    # first_mb_in_slice
    bs.ue(7)                    # slice_type I (all slices)
    bs.ue(0)                    # pic_parameter_set_id
    bs.u(0, 4)                  # frame_num
    bs.ue(idr_pic_id)
    bs.u(0, 1)                  # no_output_of_prior_pics_flag
    bs.u(0, 1)                  # long_term_reference_flag
    bs.se(0)                    # slice_qp_delta
    for my in range(mh):
        for mx in range(mw):
            x0, y0 = 16 * mx, 16 * my
            src = y[y0:y0 + 16, x0:x0 + 16]
            preds = pred_modes(ry, x0, y0, 16, False)
            mode = min(preds, key=lambda m: (satd(src - preds[m]), m))
            dcl, acl, rec = code_plane(src, preds[mode], qp, False)
            ry[y0:y0 + 16, x0:x0 + 16] = rec
            cx0, cy0 = 8 * mx, 8 * my
            srcs = (cb[cy0:cy0 + 8, cx0:cx0 + 8], cr[cy0:cy0 + 8, cx0:cx0 + 8])
            cpreds = [pred_modes(p, cx0, cy0, 8, True) for p in (rcb, rcr)]
            cmode = min(cpreds[0], key=lambda m: (satd(srcs[0] - cpreds[0][m]) + satd(srcs[1] - cpreds[1][m]), m))
            cres = []
            for c, rp in enumerate((rcb, rcr)):
                cdcl, cacl, crec = code_plane(srcs[c], cpreds[c][cmode], qpc, True)
                rp[cy0:cy0 + 8, cx0:cx0 + 8] = crec
                cres.append((cdcl, cacl))
            cbp_l = 15 if np.any(acl) else 0
            cbp_c = 2 if any(np.any(a) for _, a in cres) else 1 if any(np.any(d) for d, _ in cres) else 0
            bs.ue(1 + mode + 4 * cbp_c + (12 if cbp_l else 0))      # mb_type I_16x16_<mode>_<cbp_c>_<cbp_l>
            bs.ue(cmode)                                            # intra_chroma_pred_mode
            bs.se(0)                                                # mb_qp_delta
            gx, gy = 4 * mx, 4 * my
            residual_block(bs, dcl.reshape(16)[ZIGZAG], nc_of(tcy, gy, gx), 16)
            for b8 in range(4):
                for b4 in range(4):
                    bx, by = 2 * (b8 & 1) + (b4 & 1), 2 * (b8 >> 1) + (b4 >> 1)
                    t = 0
                    if cbp_l:
                        t = residual_block(bs, acl[by, bx][ZIGZAG][1:], nc_of(tcy, gy + by, gx + bx), 15)
                    tcy[gy + by, gx + bx] = t
            if cbp_c:
                for c in range(2):
                    residual_block(bs, cres[c][0].reshape(4), -1, 4)
            for c in range(2):
                for b in range(4):
                    bx, by = b & 1, b >> 1
                    t = 0
                    if cbp_c == 2:
                        t = residual_block(bs, cres[c][1][by, bx][ZIGZAG][1:], nc_of(tcc[c], 2 * my + by, 2 * mx + bx), 15)
                    tcc[c, 2 * my + by, 2 * mx + bx] = t
    bs.trailing()
    return nal(0x65, bs.bytes()), (ry, rcb, rcr)


def sps_pps(h, w, qp, fps):
    """(SPS, PPS) NAL units (no start code or length) for frames h x w at `fps` and `qp`"""
    mw, mh = (w + 15) // 16, (h + 15) // 16
    s = Bits()
    s.u(66, 8)
    s.u(0b11000000, 8)          # constraint_set0_flag, constraint_set1_flag
    s.u(level_idc(h, w, fps), 8)
    s.ue(0)                     # seq_parameter_set_id
    s.ue(0)                     # log2_max_frame_num_minus4
    s.ue(2)                     # pic_order_cnt_type
    s.ue(0)                     # max_num_ref_frames
    s.u(0, 1)                   # gaps_in_frame_num_value_allowed_flag
    s.ue(mw - 1)
    s.ue(mh - 1)
    s.u(1, 1)                   # frame_mbs_only_flag
    s.u(1, 1)                   # direct_8x8_inference_flag
    crop = (16 * mw != w) or (16 * mh != h)
    s.u(int(crop), 1)
    if crop:
        s.ue(0)
        s.ue((16 * mw - w) // 2)
        s.ue(0)
        s.ue((16 * mh - h) // 2)
    s.u(1, 1)                   # vui_parameters_present_flag
    s.u(1, 1)                   # aspect_ratio_info_present_flag
    s.u(1, 8)                   # aspect_ratio_idc 1:1
    s.u(0, 1)                   # overscan_info_present_flag
    s.u(1, 1)                   # video_signal_type_present_flag
    s.u(5, 3)                   # video_format unspecified
    s.u(0, 1)                   # video_full_range_flag
    s.u(1, 1)                   # colour_description_present_flag
    s.u(6, 8)
    s.u(6, 8)
    s.u(6, 8)
    s.u(0, 1)                   # chroma_loc_info_present_flag
    s.u(0, 1)                   # timing_info_present_flag
    s.u(0, 1)                   # nal_hrd_parameters_present_flag
    s.u(0, 1)                   # vcl_hrd_parameters_present_flag
    s.u(0, 1)                   # pic_struct_present_flag
    s.u(1, 1)                   # bitstream_restriction_flag
    s.u(1, 1)                   # motion_vectors_over_pic_boundaries_flag
    s.ue(0)                     # max_bytes_per_pic_denom
    s.ue(0)                     # max_bits_per_mb_denom
    s.ue(0)                     # log2_max_mv_length_horizontal
    s.ue(0)                     # log2_max_mv_length_vertical
    s.ue(0)                     # max_num_reorder_frames
    s.ue(0)                     # max_dec_frame_buffering
    s.trailing()
    p = Bits()
    p.ue(0)                     # pic_parameter_set_id
    p.ue(0)                     # seq_parameter_set_id
    p.u(0, 1)                   # entropy_coding_mode_flag
    p.u(0, 1)                   # bottom_field_pic_order_in_frame_present_flag
    p.ue(0)                     # num_slice_groups_minus1
    p.ue(0)
    p.ue(0)                     # num_ref_idx_l0 / l1_default_active_minus1
    p.u(0, 1)                   # weighted_pred_flag
    p.u(0, 2)                   # weighted_bipred_idc
    p.se(qp - 26)               # pic_init_qp_minus26
    p.se(0)                     # pic_init_qs_minus26
    p.se(0)                     # chroma_qp_index_offset
    p.u(0, 1)                   # deblocking_filter_control_present_flag
    p.u(0, 1)                   # constrained_intra_pred_flag
    p.u(0, 1)                   # redundant_pic_cnt_present_flag
    p.trailing()
    return nal(0x67, s.bytes()), nal(0x68, p.bytes())


def encode(frames, qp, fps=30, first_frame=0):
    """(sps, pps, [access unit]) of u8 RGB frames [n, h, w, 3]: each access unit its IDR slice NAL unit with a 4-byte big-endian
    length prefix (the MP4 sample); frame i's idr_pic_id is (first_frame + i) & 1"""
    frames = np.asarray(frames)
    n, h, w, _ = frames.shape
    check_args(h, w, qp)
    sps, pps = sps_pps(h, w, qp, fps)
    aus = []
    for i in range(n):
        s, _ = encode_picture(frames[i], qp, (first_frame + i) & 1)
        aus.append(len(s).to_bytes(4, 'big') + s)
    return sps, pps, aus


# ------------------------------------------------------------------------------------------------ decoder side
def _filter_edge(p, q, bs, alpha, beta, tc0, chroma):
    """8.7.2.3 / 8.7.2.4 on sample lines p[k], q[k] ([3 or 4, L] arrays, k = distance from the edge - 1); returns (p', q')"""
    p, q = p.copy(), q.copy()
    p0, p1, q0, q1 = p[0].copy(), p[1].copy(), q[0].copy(), q[1].copy()
    on = (np.abs(p0 - q0) < alpha) & (np.abs(p1 - p0) < beta) & (np.abs(q1 - q0) < beta)
    if chroma:
        if bs == 4:
            np0 = (2 * p1 + p0 + q1 + 2) >> 2
            nq0 = (2 * q1 + q0 + p1 + 2) >> 2
        else:
            tc = tc0 + 1
            delta = np.clip((((q0 - p0) << 2) + (p1 - q1) + 4) >> 3, -tc, tc)
            np0, nq0 = np.clip(p0 + delta, 0, 255), np.clip(q0 - delta, 0, 255)
        p[0] = np.where(on, np0, p0)
        q[0] = np.where(on, nq0, q0)
        return p, q
    p2, q2 = p[2].copy(), q[2].copy()
    ap, aq = np.abs(p2 - p0), np.abs(q2 - q0)
    if bs == 4:
        p3, q3 = p[3].copy(), q[3].copy()
        strong = (np.abs(p0 - q0) < ((alpha >> 2) + 2))
        sp, sq = on & (ap < beta) & strong, on & (aq < beta) & strong
        new_p = [np.where(sp, (p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3, (2 * p1 + p0 + q1 + 2) >> 2),
                 (p2 + p1 + p0 + q0 + 2) >> 2, (2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3]
        new_q = [np.where(sq, (p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3, (2 * q1 + q0 + p1 + 2) >> 2),
                 (p0 + q0 + q1 + q2 + 2) >> 2, (2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3]
        p[0] = np.where(on, new_p[0], p0)
        q[0] = np.where(on, new_q[0], q0)
        p[1] = np.where(sp, new_p[1], p1)
        q[1] = np.where(sq, new_q[1], q1)
        p[2] = np.where(sp, new_p[2], p2)
        q[2] = np.where(sq, new_q[2], q2)
        return p, q
    tc = tc0 + (ap < beta) + (aq < beta)
    delta = np.clip((((q0 - p0) << 2) + (p1 - q1) + 4) >> 3, -tc, tc)
    p[0] = np.where(on, np.clip(p0 + delta, 0, 255), p0)
    q[0] = np.where(on, np.clip(q0 - delta, 0, 255), q0)
    avg = (p0 + q0 + 1) >> 1
    p[1] = np.where(on & (ap < beta), p1 + np.clip((p2 + avg - (p1 << 1)) >> 1, -tc0, tc0), p1)
    q[1] = np.where(on & (aq < beta), q1 + np.clip((q2 + avg - (q1 << 1)) >> 1, -tc0, tc0), q1)
    return p, q


def deblock(planes, qp):
    """the decoder's loop filter (8.7) over padded reconstruction planes of an all-intra single-slice picture: bS 4 on macroblock
    edges inside the picture, 3 on inner 4x4 edges; macroblocks in raster order, vertical edges then horizontal, luma then chroma"""
    out = [p.astype(np.int64).copy() for p in planes]
    for c, pl in enumerate(out):
        chroma = c > 0
        q = QPC[qp] if chroma else qp
        alpha, beta, tc0 = ALPHA[q], BETA[q], TC0_BS3[q]
        n = 8 if chroma else 16
        depth = 2 if chroma else 4
        mh, mw = pl.shape[0] // n, pl.shape[1] // n
        edges = (0, 4) if chroma else (0, 4, 8, 12)
        for my in range(mh):
            for mx in range(mw):
                x0, y0 = n * mx, n * my
                for vertical in (True, False):
                    for e in edges:
                        if e == 0 and (mx if vertical else my) == 0:
                            continue
                        bs = 4 if e == 0 else 3
                        if vertical:
                            xs = x0 + e
                            pp = pl[y0:y0 + n, xs - depth:xs][:, ::-1].T
                            qq = pl[y0:y0 + n, xs:xs + depth].T
                            np_, nq = _filter_edge(pp, qq, bs, alpha, beta, tc0, chroma)
                            pl[y0:y0 + n, xs - depth:xs] = np_[::-1].T
                            pl[y0:y0 + n, xs:xs + depth] = nq.T
                        else:
                            ys = y0 + e
                            pp = pl[ys - depth:ys, x0:x0 + n][::-1]
                            qq = pl[ys:ys + depth, x0:x0 + n]
                            np_, nq = _filter_edge(pp, qq, bs, alpha, beta, tc0, chroma)
                            pl[ys - depth:ys, x0:x0 + n] = np_[::-1]
                            pl[ys:ys + depth, x0:x0 + n] = nq
    return out


def decoded_planes(frame, qp, idr_pic_id=0):
    """the decoder's output (Y [h, w], Cb, Cr [h / 2, w / 2]) u8 for one u8 RGB frame: deblocked reconstruction, cropped"""
    h, w, _ = frame.shape
    _, rec = encode_picture(frame, qp, idr_pic_id)
    y, cb, cr = deblock(rec, qp)
    return y[:h, :w].astype(np.uint8), cb[:h // 2, :w // 2].astype(np.uint8), cr[:h // 2, :w // 2].astype(np.uint8)


def annexb(sps, pps, aus):
    """an Annex B byte stream (start codes) of the SPS, PPS and length-prefixed access units"""
    out = b'\0\0\0\1' + sps + b'\0\0\0\1' + pps
    for au in aus:
        k = 0
        while k < len(au):
            ln = int.from_bytes(au[k:k + 4], 'big')
            out += b'\0\0\0\1' + au[k + 4:k + 4 + ln]
            k += 4 + ln
    return out
