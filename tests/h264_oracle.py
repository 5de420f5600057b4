"""numpy restatement of the sm_90a H.264 encoder (next3d_b200/csrc/h264.cu): the same colour conversion, mode and motion
decisions, tie-breaks, quantisation, CAVLC, deblocking and rate control, producing the same bytes and the same reconstruction.
Test infrastructure only: the CPU tests decode its streams with FFmpeg to prove the byte format, and the GPU tests compare the
kernels with it byte for byte.  The parameter sets (SPS / PPS) come from next3d_b200.video, which writes them for both encoders.

Stream subset (see DESIGN.md section 3.5): Constrained Baseline, one slice per macroblock row, IDR frames of I_16x16 macroblocks
(DC or horizontal luma prediction, DC chroma), P frames of P_L0_16x16 / P_Skip.  Two streams, as the kernels' kRc parameter:
- `Encoder` (n3d_h264_encode): constant QP (pic_init_qp = QP), integer-pel motion, no deblocking.
- `RcEncoder` (n3d_h264_encode_rc): pic_init_qp 26 with slice_qp_delta = QP - 26 (one QP per picture, chosen by the controller
  before the picture is coded), vectors refined to quarter samples around the integer search's best vector, and
  disable_deblocking_filter_idc 0 (the deblocked picture is the output and the next P frame's reference)."""
import re

import numpy as np

SEARCH = 16                     # integer-pel full search over [-SEARCH, SEARCH]^2 (csrc/h264.cu kSearch)
PAD = SEARCH + 8                # reference padding: covers the search, the quarter-sample refinement and the 6-tap filter
MV_OFF = 128                    # key offset of quarter-sample vector components (|mv| <= 4 * SEARCH + 3)
LEVEL_MAX = 2063                # largest |level| CAVLC codes with level_prefix <= 15 at every suffixLength (Baseline)

LAMBDA = [0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 5, 5, 6, 7, 7, 8, 9, 10, 12, 13, 15,
          17, 19, 21, 23, 26, 30, 33, 37, 42, 47, 53, 59, 66, 74, 83]
QPC = list(range(30)) + [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39]
MF = [[13107, 5243, 8066], [11916, 4660, 7490], [10082, 4194, 6554], [9362, 3647, 5825], [8192, 3355, 5243], [7282, 2893, 4559]]
V = [[10, 16, 13], [11, 18, 14], [13, 20, 16], [14, 23, 18], [16, 25, 20], [18, 29, 23]]
ZZ = [0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15]               # frame zig-zag scan -> raster index in a 4x4 block
BLK = [(0, 0), (1, 0), (0, 1), (1, 1), (2, 0), (3, 0), (2, 1), (3, 1),   # luma4x4BlkIdx -> (x, y) in 4x4 units
       (0, 2), (1, 2), (0, 3), (1, 3), (2, 2), (3, 2), (2, 3), (3, 3)]
INTER_CBP = [0, 16, 1, 2, 4, 8, 32, 3, 5, 10, 12, 15, 47, 7, 11, 13, 14, 6, 9, 31, 35, 37, 42, 44, 33, 34, 36, 40, 39, 43, 45, 46,
             17, 18, 20, 24, 19, 21, 26, 28, 23, 27, 29, 30, 22, 25, 38, 41]          # me(v) codeNum -> inter coded_block_pattern
CBP_CODE = {c: k for k, c in enumerate(INTER_CBP)}

# coeff_token (Table 9-5), index 4 * TotalCoeff + TrailingOnes, for 0 <= nC < 2, 2 <= nC < 4, 4 <= nC < 8, 8 <= nC
CT_LEN = [
    [1, 0, 0, 0, 6, 2, 0, 0, 8, 6, 3, 0, 9, 8, 7, 5, 10, 9, 8, 6, 11, 10, 9, 7, 13, 11, 10, 8, 13, 13, 11, 9, 13, 13, 13, 10,
     14, 14, 13, 11, 14, 14, 14, 13, 15, 15, 14, 14, 15, 15, 15, 14, 16, 15, 15, 15, 16, 16, 16, 15, 16, 16, 16, 16, 16, 16, 16, 16],
    [2, 0, 0, 0, 6, 2, 0, 0, 6, 5, 3, 0, 7, 6, 6, 4, 8, 6, 6, 4, 8, 7, 7, 5, 9, 8, 8, 6, 11, 9, 9, 6, 11, 11, 11, 7,
     12, 11, 11, 9, 12, 12, 12, 11, 12, 12, 12, 11, 13, 13, 13, 12, 13, 13, 13, 13, 13, 14, 13, 13, 14, 14, 14, 13, 14, 14, 14, 14],
    [4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4, 7, 5, 5, 4, 7, 5, 5, 4, 7, 6, 6, 4, 7, 6, 6, 4, 8, 7, 7, 5,
     8, 8, 7, 6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10],
    [6, 0, 0, 0] + [6] * 64,
]
CT_BITS = [
    [1, 0, 0, 0, 5, 1, 0, 0, 7, 4, 1, 0, 7, 6, 5, 3, 7, 6, 5, 3, 7, 6, 5, 4, 15, 6, 5, 4, 11, 14, 5, 4, 8, 10, 13, 4,
     15, 14, 9, 4, 11, 10, 13, 12, 15, 14, 9, 12, 11, 10, 13, 8, 15, 1, 9, 12, 11, 14, 13, 8, 7, 10, 9, 12, 4, 6, 5, 8],
    [3, 0, 0, 0, 11, 2, 0, 0, 7, 7, 3, 0, 7, 10, 9, 5, 7, 6, 5, 4, 4, 6, 5, 6, 7, 6, 5, 8, 15, 6, 5, 4, 11, 14, 13, 4,
     15, 10, 9, 4, 11, 14, 13, 12, 8, 10, 9, 8, 15, 14, 13, 12, 11, 10, 9, 12, 7, 11, 6, 8, 9, 8, 10, 1, 7, 6, 5, 4],
    [15, 0, 0, 0, 15, 14, 0, 0, 11, 15, 13, 0, 8, 12, 14, 12, 15, 10, 11, 11, 11, 8, 9, 10, 9, 14, 13, 9, 8, 10, 9, 8,
     15, 14, 13, 13, 11, 14, 10, 12, 15, 10, 13, 12, 11, 14, 9, 12, 8, 10, 13, 8, 13, 7, 9, 12, 9, 12, 11, 10, 5, 8, 7, 6,
     1, 4, 3, 2],
    [3, 0, 0, 0, 0, 1, 0, 0, 4, 5, 6, 0] + list(range(8, 64)),
]
CDC_CT_LEN = [2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7]            # chroma DC (nC = -1)
CDC_CT_BITS = [1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0]
TZ_LEN = [[1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9], [3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6], [4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6],
          [5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5], [4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5], [6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6],
          [6, 5, 3, 3, 3, 2, 3, 4, 3, 6], [6, 4, 5, 3, 2, 2, 3, 3, 6], [6, 6, 4, 2, 2, 3, 2, 5], [5, 5, 3, 2, 2, 2, 4], [4, 4, 3, 3, 1, 3],
          [4, 4, 2, 1, 3], [3, 3, 1, 2], [2, 2, 1], [1, 1]]
TZ_BITS = [[1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1], [7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0], [5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0],
           [3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0], [5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0],
           [1, 1, 5, 4, 3, 3, 2, 1, 1, 0], [1, 1, 1, 3, 3, 2, 2, 1, 0], [1, 0, 1, 3, 2, 1, 1, 1], [1, 0, 1, 3, 2, 1, 1], [0, 1, 1, 2, 1, 3],
           [0, 1, 1, 1, 1], [0, 1, 1, 1], [0, 1, 1], [0, 1]]
CDC_TZ_LEN = [[1, 2, 3, 3], [1, 2, 2], [1, 1]]
CDC_TZ_BITS = [[1, 1, 1, 0], [1, 1, 0], [1, 0]]
RUN_LEN = [[1, 1], [1, 2, 2], [2, 2, 2, 2], [2, 2, 2, 3, 3], [2, 2, 3, 3, 3, 3], [2, 3, 3, 3, 3, 3, 3],
           [3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11]]
RUN_BITS = [[1, 0], [1, 1, 0], [3, 2, 1, 0], [3, 2, 1, 1, 0], [3, 2, 3, 2, 1, 0], [3, 0, 1, 3, 2, 5, 4],
            [7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1]]

CF = np.array([[1, 1, 1, 1], [2, 1, -1, -2], [1, -1, -1, 1], [1, -2, 2, -1]], np.int64)
HAD = np.array([[1, 1, 1, 1], [1, 1, -1, -1], [1, -1, -1, 1], [1, -1, 1, -1]], np.int64)
A2 = np.array([[1, 1], [1, -1]], np.int64)


def _cls4():
    c = np.full((4, 4), 2)
    c[0::2, 0::2] = 0
    c[1::2, 1::2] = 1
    return c


CLS = _cls4()
MF4 = np.array([np.array(m)[CLS] for m in MF], np.int64)        # [qp % 6, 4, 4]
LS4 = np.array([16 * np.array(v)[CLS] for v in V], np.int64)    # LevelScale4x4 with flat weights


# ------------------------------------------------------------------------------------------------ colour conversion
def rgb_to_yuv420(rgb):
    """uint8 RGB [H, W, 3] (H, W even) -> padded Y [H16, W16], Cb, Cr [H16/2, W16/2] uint8, BT.601 limited range in integers;
    the padding repeats the last row / column of each plane."""
    H, W, _ = rgb.shape
    x = rgb.astype(np.int64)
    R, G, B = x[..., 0], x[..., 1], x[..., 2]
    y = ((66 * R + 129 * G + 25 * B + 128) >> 8) + 16
    s = lambda p: p[0::2, 0::2] + p[1::2, 0::2] + p[0::2, 1::2] + p[1::2, 1::2]
    sR, sG, sB = s(R), s(G), s(B)
    cb = ((-38 * sR - 74 * sG + 112 * sB + 512) >> 10) + 128
    cr = ((112 * sR - 94 * sG - 18 * sB + 512) >> 10) + 128
    H16, W16 = (H + 15) // 16 * 16, (W + 15) // 16 * 16
    pad = lambda p, h, w: np.pad(p, ((0, h - p.shape[0]), (0, w - p.shape[1])), mode='edge').astype(np.uint8)
    return pad(y, H16, W16), pad(cb, H16 // 2, W16 // 2), pad(cr, H16 // 2, W16 // 2)


# ------------------------------------------------------------------------------------------------ transforms and quantisation
def fwd4(x):
    return CF @ x @ CF.T


def inv4(d):
    """8.5.12.2 on [..., 4, 4] scaled coefficients, then (x + 32) >> 6."""
    d = d.astype(np.int64)

    def one(a):                               # 1-D inverse along the last axis
        e0, e1 = a[..., 0] + a[..., 2], a[..., 0] - a[..., 2]
        e2, e3 = (a[..., 1] >> 1) - a[..., 3], a[..., 1] + (a[..., 3] >> 1)
        return np.stack([e0 + e3, e1 + e2, e1 - e2, e0 - e3], -1)
    f = one(d)
    h = np.swapaxes(one(np.swapaxes(f, -1, -2)), -1, -2)
    return (h + 32) >> 6


def quant(w, qp, intra, dc_shift=0, mf=None, census=None, kind=None):
    """Levels of coefficients w [..., 4, 4] (or of a DC transform); census (a Counter, or None) counts the levels of this block
    kind clamped to LEVEL_MAX (for an AC kind, outside the DC position, whose level the caller drops)."""
    qbits = 15 + qp // 6 + dc_shift
    f = ((1 << (15 + qp // 6)) // (3 if intra else 6)) << dc_shift
    mf = MF4[qp % 6] if mf is None else mf
    lv = (np.abs(w) * mf + f) >> qbits
    if census is not None:
        over = lv > LEVEL_MAX
        if kind.endswith('AC'):
            over[..., 0, 0] = False
        census['clamp', kind] += int(over.sum())
    return (np.sign(w) * np.minimum(lv, LEVEL_MAX)).astype(np.int64)


def dequant(c, qp):
    ls = LS4[qp % 6]
    if qp >= 24:
        return (c * ls) << (qp // 6 - 4)
    return (c * ls + (1 << (3 - qp // 6))) >> (4 - qp // 6)


def blocks(mb):
    """[..., 16, 16] macroblock -> [..., 16, 4, 4] in luma4x4BlkIdx order."""
    return np.stack([mb[..., 4 * by:4 * by + 4, 4 * bx:4 * bx + 4] for bx, by in BLK], -3)


def unblocks(b):
    out = np.zeros(b.shape[:-3] + (16, 16), b.dtype)
    for k, (bx, by) in enumerate(BLK):
        out[..., 4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = b[..., k, :, :]
    return out


def cblocks(mb):
    """[..., 8, 8] chroma macroblock -> [..., 4, 4, 4] in raster block order."""
    return np.stack([mb[..., 4 * by:4 * by + 4, 4 * bx:4 * bx + 4] for by in range(2) for bx in range(2)], -3)


def uncblocks(b):
    out = np.zeros(b.shape[:-3] + (8, 8), b.dtype)
    for k in range(4):
        by, bx = divmod(k, 2)
        out[..., 4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = b[..., k, :, :]
    return out


def scan(b):
    """[..., 4, 4] -> [..., 16] in zig-zag order."""
    return b.reshape(b.shape[:-2] + (16,))[..., ZZ]


def code_chroma(src, pred, qpc, intra, census=None):
    """One chroma component of a batch of macroblocks: src, pred [..., 8, 8] -> (DC levels [..., 4], AC levels [..., 4, 16] in
    zig-zag order (index 0 unused), reconstruction [..., 8, 8])."""
    frame = 'I' if intra else 'P'
    w = fwd4(cblocks(src.astype(np.int64) - pred))
    dc = w[..., 0, 0]
    t = np.einsum('ij,...jk,kl->...il', A2, dc.reshape(dc.shape[:-1] + (2, 2)), A2)
    dcl = quant(t, qpc, intra, 1, MF4[qpc % 6][0, 0], census, f'{frame} chroma DC').reshape(dc.shape)
    acl = quant(w, qpc, intra, census=census, kind=f'{frame} chroma AC')
    acl[..., 0, 0] = 0
    f = np.einsum('ij,...jk,kl->...il', A2, dcl.reshape(dcl.shape[:-1] + (2, 2)), A2)
    dcc = ((f * LS4[qpc % 6][0, 0]) << (qpc // 6)) >> 5
    d = dequant(acl, qpc)
    d[..., 0, 0] = dcc.reshape(dc.shape)
    rec = np.clip(pred + uncblocks(inv4(d)), 0, 255)
    return dcl, scan(acl), rec


# ------------------------------------------------------------------------------------------------ bit writing
def se_code(v):
    return 2 * v - 1 if v > 0 else -2 * v


def se_bits(v):
    """Length of se(v) for an array of values."""
    k = np.where(v > 0, 2 * v - 1, -2 * v)
    return 2 * np.frexp(k + 1.0)[1].astype(np.int64) - 1


class Bits:
    def __init__(self, census=None):
        self.parts = []
        self.census = census                  # a Counter of the CAVLC syntax written (residual_block), or None

    def u(self, v, n):
        if n:
            self.parts.append(format(int(v), f'0{n}b'))

    def ue(self, k):
        n = (int(k) + 1).bit_length()
        self.u(0, n - 1)
        self.u(k + 1, n)

    def se(self, v):
        self.ue(se_code(int(v)))

    def rbsp(self):
        """Bits + rbsp_trailing_bits -> bytes."""
        s = ''.join(self.parts) + '1'
        s += '0' * (-len(s) % 8)
        return int(s, 2).to_bytes(len(s) // 8, 'big')


def escape(rbsp):
    """Emulation prevention: 0x000003 before any 0x0000xx with xx <= 3."""
    return re.sub(b'\x00\x00(?=[\x00-\x03])', b'\x00\x00\x03', rbsp)


def residual_block(bw, coeffs, nc):
    """CAVLC residual_block (9.2) of coeffs (scan order, len 16, 15 or 4); nc = -1 for chroma DC.  Returns TotalCoeff."""
    coeffs = [int(c) for c in coeffs]
    nz = [i for i, c in enumerate(coeffs) if c]
    total = len(nz)
    t1 = 0
    for i in reversed(nz):
        if abs(coeffs[i]) != 1 or t1 == 3:
            break
        t1 += 1
    idx = 4 * total + t1
    rec = bw.census
    if nc == -1:
        bw.u(CDC_CT_BITS[idx], CDC_CT_LEN[idx])
    else:
        tab = 0 if nc < 2 else 1 if nc < 4 else 2 if nc < 8 else 3
        bw.u(CT_BITS[tab][idx], CT_LEN[tab][idx])
    if rec is not None:
        rec['coeff_token', 'chroma DC' if nc == -1 else ('nC 0-1', 'nC 2-3', 'nC 4-7', 'nC >= 8')[tab]] += 1
        if nc != -1 and total:
            rec['TotalCoeff', total] += 1
    if total == 0:
        return 0
    levels = [coeffs[i] for i in reversed(nz)]
    for k in range(t1):
        bw.u(1 if levels[k] < 0 else 0, 1)
    sl = 1 if total > 10 and t1 < 3 else 0
    for k in range(t1, total):
        lv = levels[k]
        code = 2 * lv - 2 if lv > 0 else -2 * lv - 1
        if k == t1 and t1 < 3:
            code -= 2
        if sl == 0:
            if code < 14:
                prefix, sbits, sval = code, 0, 0
            elif code < 30:
                prefix, sbits, sval = 14, 4, code - 14
            else:
                prefix, sbits, sval = 15, 12, code - 30
        elif code < (15 << sl):
            prefix, sbits, sval = code >> sl, sl, code & ((1 << sl) - 1)
        else:
            prefix, sbits, sval = 15, 12, code - (15 << sl)
        bw.u(1, prefix + 1)
        bw.u(sval, sbits)
        if rec is not None:
            rec['level_prefix', prefix] += 1
            rec['suffixLength', sl] += 1
        if sl == 0:
            sl = 1
        if abs(lv) > (3 << (sl - 1)) and sl < 6:
            sl += 1
    n = len(coeffs)
    if total < n:
        tz = nz[-1] + 1 - total
        if rec is not None:
            rec['total_zeros', 'chroma DC' if nc == -1 else '4x4', total] += 1
            rec['total_zeros pair', 'chroma DC' if nc == -1 else '4x4', total, tz] += 1
        if nc == -1:
            bw.u(CDC_TZ_BITS[total - 1][tz], CDC_TZ_LEN[total - 1][tz])
        else:
            bw.u(TZ_BITS[total - 1][tz], TZ_LEN[total - 1][tz])
        left = tz
        for j in range(total - 1, 0, -1):
            if left == 0:
                break
            run = nz[j] - nz[j - 1] - 1
            t = min(left, 7) - 1
            bw.u(RUN_BITS[t][run], RUN_LEN[t][run])
            if rec is not None:
                rec['run_before', 'zerosLeft > 6' if t == 6 else f'zerosLeft {t + 1}'] += 1
            left -= run
    return total


def _nc(na, nb):
    """nC of coeff_token (9.2.1) from the left / upper block's TotalCoeff, None when that block is not available."""
    if na is not None and nb is not None:
        return (na + nb + 1) >> 1
    return na if na is not None else nb if nb is not None else 0


# ------------------------------------------------------------------------------------------------ encoder
def _mb_view(p, s):
    """[R*s, C*s] plane -> [R, C, s, s] macroblock view."""
    R, C = p.shape[0] // s, p.shape[1] // s
    return p.reshape(R, s, C, s).swapaxes(1, 2)


def mv_key(cost, qx, qy):
    """Search key of a vector (qx, qy) in quarter samples: the smallest key has the smallest cost, then the smallest |mv|_1, then
    the smallest (mvy, mvx) (csrc/h264.cu mv_key)."""
    return (cost << 24) | ((np.abs(qx) + np.abs(qy)) << 16) | ((qy + MV_OFF) << 8) | (qx + MV_OFF)


def mv_of(key):
    """(qx, qy) of mv_key keys."""
    return (key & 0xff) - MV_OFF, ((key >> 8) & 0xff) - MV_OFF


class Encoder:
    """The constant-QP stream: encodes uint8 RGB frames into length-prefixed slice NAL units, one sample per frame.  The first
    frame and every gop-th one after it is IDR."""

    census = None                             # a Counter of the syntax and decisions of every frame encoded, or None (see record())

    def __init__(self, width, height, qp=18, gop=60):
        if width % 2 or height % 2 or width <= 0 or height <= 0:
            raise ValueError('4:2:0 needs even, positive frame dimensions')
        self.W, self.H, self.qp, self.gop = width, height, qp, gop
        self.mbw, self.mbh = (width + 15) // 16, (height + 15) // 16
        self.n = 0
        self.recon = None                     # (Y, Cb, Cr) padded planes of the last frame
        self.mvs = None                       # [mbh, mbw, 2] MVs of the last P frame in quarter samples
        self.skip = None                      # [mbh, mbw] bool
        self.levels = None                    # [mbh, mbw, 16, 4, 4] luma levels of the last P frame (luma4x4BlkIdx order)

    # ---------------------------------------------------------------- decisions and reconstruction
    def _intra(self, Y, U, V):
        """I_16x16 for every MB; column by column (each MB needs its left neighbour's reconstruction), rows at once."""
        qp, qpc = self.qp, QPC[self.qp]
        R, C = self.mbh, self.mbw
        yb, ub, vb = _mb_view(Y.astype(np.int64), 16), _mb_view(U.astype(np.int64), 8), _mb_view(V.astype(np.int64), 8)
        ry, ru, rv = np.zeros_like(yb), np.zeros_like(ub), np.zeros_like(vb)
        mbs = [[None] * C for _ in range(R)]
        for c in range(C):
            src = yb[:, c]
            if c == 0:
                pred = np.full_like(src, 128)
                mode = np.full(R, 2)
            else:
                left = ry[:, c - 1, :, 15]                                     # [R, 16]
                dcp = ((left.sum(-1) + 8) >> 4)[:, None, None] * np.ones((1, 16, 16), np.int64)
                hp = np.repeat(left[:, :, None], 16, -1)
                sad_h = np.abs(src - hp).sum((-1, -2))
                sad_dc = np.abs(src - dcp).sum((-1, -2))
                useh = sad_h <= sad_dc
                pred = np.where(useh[:, None, None], hp, dcp)
                mode = np.where(useh, 1, 2)
            w = fwd4(blocks(src - pred))                                     # [R, 16, 4, 4]
            dcm = unblocks_dc(w[..., 0, 0])                                  # [R, 4, 4] spatial
            hd = (HAD @ dcm @ HAD) >> 1
            dcl = quant(hd, qp, True, 1, MF4[qp % 6][0, 0], self.census, 'I luma DC')
            acl = quant(w, qp, True, census=self.census, kind='I luma AC')
            acl[..., 0, 0] = 0
            c4 = HAD @ dcl @ HAD
            if qp >= 36:
                dcy = (c4 * LS4[qp % 6][0, 0]) << (qp // 6 - 6)
            else:
                dcy = (c4 * LS4[qp % 6][0, 0] + (1 << (5 - qp // 6))) >> (6 - qp // 6)
            d = dequant(acl, qp)
            d[..., 0, 0] = blocks_dc(dcy)
            ry[:, c] = np.clip(pred + unblocks(inv4(d)), 0, 255)
            cres = []
            for comp, (sb, rb) in enumerate(((ub, ru), (vb, rv))):
                if c == 0:
                    cp = np.full((R, 8, 8), 128, np.int64)
                else:
                    lc = rb[:, c - 1, :, 7]                                      # [R, 8]
                    top = (lc[:, 0:4].sum(-1) + 2) >> 2
                    bot = (lc[:, 4:8].sum(-1) + 2) >> 2
                    cp = np.concatenate([np.repeat(top[:, None, None], 4, 1), np.repeat(bot[:, None, None], 4, 1)], 1)
                    cp = np.repeat(cp, 8, -1)
                dcl_c, acl_c, rec_c = code_chroma(sb[:, c], cp, qpc, True, self.census)
                rb[:, c] = rec_c
                cres.append((dcl_c, acl_c))
            for r in range(R):
                mbs[r][c] = dict(intra=True, mode=int(mode[r]), ldc=scan(dcl[r]), lac=scan(acl[r]),
                                 cdc=[cres[0][0][r], cres[1][0][r]], cac=[cres[0][1][r], cres[1][1][r]])
        return mbs, (ry, ru, rv)

    def _integer_search(self, G, cur):
        """Integer-pel full search over [-SEARCH, SEARCH]^2 of every MB of cur [H16, W16] against G, the reference luma padded by
        PAD with its edge samples (the decoder's clamped coordinates).  cost = SAD + lambda * bits of the MV against a zero
        predictor (so that MBs are decided independently).  Returns the best mv_key per MB [mbh, mbw]."""
        S, R, C = SEARCH, self.mbh, self.mbw
        H16, W16 = 16 * R, 16 * C
        lam = LAMBDA[self.qp]
        mx = 4 * np.arange(-S, S + 1)[:, None, None]
        G, cur = G.astype(np.int16), cur.astype(np.int16)           # differences of samples fit: 4x less memory than int64
        best = np.full((R, C), np.iinfo(np.int64).max, np.int64)
        for my in range(-S, S + 1):                   # all mx at once
            rows = G[PAD + my:PAD + my + H16, PAD - S:PAD + S + W16]
            shifted = np.lib.stride_tricks.sliding_window_view(rows, W16, 1).swapaxes(0, 1)              # [mx, H16, W16]
            sad = np.abs(cur - shifted).reshape(2 * S + 1, R, 16, C, 16).sum((2, 4), dtype=np.int64)
            cost = sad + lam * (se_bits(mx) + se_bits(4 * my))
            np.minimum(best, mv_key(cost, mx, 4 * my).min(0), out=best)
        return best

    def _search(self, ry, cur):
        """Motion search of every MB against the reference luma ry: (mvx, mvy [mbh, mbw] in quarter samples, luma prediction
        [mbh, mbw, 16, 16])."""
        G = np.pad(ry, PAD, mode='edge')
        qx, qy = mv_of(self._integer_search(G, cur))
        R, C = self.mbh, self.mbw
        yy = PAD + 16 * np.arange(R)[:, None, None, None] + np.arange(16)[None, None, :, None] + (qy >> 2)[:, :, None, None]
        xx = PAD + 16 * np.arange(C)[None, :, None, None] + np.arange(16)[None, None, None, :] + (qx >> 2)[:, :, None, None]
        return qx, qy, G[yy, xx]

    def _inter(self, Y, U, V):
        """P_L0_16x16 / P_Skip for every MB at once against the previous reconstruction."""
        qp, qpc = self.qp, QPC[self.qp]
        R, C = self.mbh, self.mbw
        H16, W16 = 16 * R, 16 * C
        ry, ru, rv = (p.astype(np.int64) for p in self.recon)
        cur = Y.astype(np.int64)
        qx, qy, pred = self._search(ry, cur)
        if self.census is not None:
            for x, y in zip((qx & 3).ravel().tolist(), (qy & 3).ravel().tolist()):
                self.census['quarter-sample position', x, y] += 1
            self.census['vector at the search bound',] += int((np.maximum(np.abs(qx), np.abs(qy)) >= 4 * SEARCH).sum())
            self.census['vector refined past the search bound',] += int((np.maximum(np.abs(qx), np.abs(qy)) > 4 * SEARCH).sum())
        w = fwd4(blocks(_mb_view(cur, 16) - pred))
        lvl = quant(w, qp, False, census=self.census, kind='P luma')          # [R, C, 16, 4, 4]
        rec_y = np.clip(pred + unblocks(inv4(dequant(lvl, qp))), 0, 255)
        # chroma: eighth-sample bilinear (8.4.2.2.2) at the luma vector, whose quarter samples are chroma eighth samples
        fx, fy = (qx & 7)[:, :, None, None], (qy & 7)[:, :, None, None]
        cy = np.arange(8)[None, None, :, None] + 8 * np.arange(R)[:, None, None, None] + (qy >> 3)[:, :, None, None]
        cx = np.arange(8)[None, None, None, :] + 8 * np.arange(C)[None, :, None, None] + (qx >> 3)[:, :, None, None]
        cres, crec = [], []
        for sp, rp in ((U, ru), (V, rv)):
            at = lambda y, x: rp[np.clip(y, 0, H16 // 2 - 1), np.clip(x, 0, W16 // 2 - 1)]
            cp = ((8 - fx) * (8 - fy) * at(cy, cx) + fx * (8 - fy) * at(cy, cx + 1) + (8 - fx) * fy * at(cy + 1, cx)
                  + fx * fy * at(cy + 1, cx + 1) + 32) >> 6
            dcl_c, acl_c, rec_c = code_chroma(_mb_view(sp.astype(np.int64), 8), cp, qpc, False, self.census)
            cres.append((dcl_c, acl_c))
            crec.append(rec_c)
        nonzero = (lvl != 0).any((-1, -2, -3)) | (cres[0][0] != 0).any(-1) | (cres[0][1] != 0).any((-1, -2)) \
            | (cres[1][0] != 0).any(-1) | (cres[1][1] != 0).any((-1, -2))
        skip = (qx == 0) & (qy == 0) & ~nonzero
        mbs = [[dict(intra=False, skip=bool(skip[r, c]), mv=(int(qx[r, c]), int(qy[r, c])), lac=scan(lvl[r, c]),
                     cdc=[cres[0][0][r, c], cres[1][0][r, c]], cac=[cres[0][1][r, c], cres[1][1][r, c]])
                for c in range(C)] for r in range(R)]
        self.mvs, self.skip, self.levels = np.stack([qx, qy], -1), skip, lvl
        return mbs, (rec_y, crec[0], crec[1])

    # ---------------------------------------------------------------- syntax
    def _slice_qp_and_deblocking(self, bw):
        """The last fields of the slice header."""
        bw.se(0)                                   # slice_qp_delta (pic_init_qp = QP)
        bw.ue(1)                                   # disable_deblocking_filter_idc

    def _slice(self, row, mbs, idr, frame_num, idr_pic_id):
        rec = self.census
        bw = Bits(rec)
        bw.ue(row * self.mbw)                      # first_mb_in_slice
        bw.ue(2 if idr else 0)                     # slice_type I / P
        bw.ue(0)                                   # pic_parameter_set_id
        bw.u(frame_num, 4)                         # log2_max_frame_num = 4
        if idr:
            bw.ue(idr_pic_id)
        else:
            bw.u(0, 1)                             # num_ref_idx_active_override_flag
            bw.u(0, 1)                             # ref_pic_list_modification_flag_l0
        bw.u(0, 1)                                 # no_output_of_prior_pics_flag / adaptive_ref_pic_marking_mode_flag
        if idr:
            bw.u(0, 1)                             # long_term_reference_flag
        self._slice_qp_and_deblocking(bw)
        left_tc = [0] * 4                          # TotalCoeff of the left MB's right-column luma blocks (rows 0..3)
        left_cc = [[0, 0], [0, 0]]                 # ... and of its right-column chroma blocks, per component
        skip_run = 0
        mvp = (0, 0)
        for c, m in enumerate(mbs):
            if not idr and m['skip']:
                skip_run += 1
                left_tc, left_cc, mvp = [0] * 4, [[0, 0], [0, 0]], (0, 0)
                continue
            tc = np.zeros((4, 4), int)             # [by, bx]
            if idr:
                nz_ac = any(np.any(m['lac'][k][1:]) for k in range(16))
                cbp_l = 15 if nz_ac else 0
            else:
                if rec is not None and skip_run:
                    rec['skip run', 'row start' if skip_run == c else 'mid-row'] += 1
                bw.ue(skip_run)
                skip_run = 0
                cbp_l = sum(1 << q for q in range(4) if any(np.any(m['lac'][4 * q + k]) for k in range(4)))
            cdc_nz = any(np.any(x) for x in m['cdc'])
            cac_nz = any(np.any(x[:, 1:]) for x in m['cac'])
            cbp_c = 2 if cac_nz else 1 if cdc_nz else 0
            if rec is not None:
                rec[('I16x16', m['mode'], cbp_c, cbp_l) if idr else ('P cbp', cbp_l, cbp_c)] += 1
            if idr:
                bw.ue(1 + m['mode'] + 4 * cbp_c + (12 if cbp_l else 0))     # mb_type I_16x16_<mode>_<cbp_c>_<cbp_l>
                bw.ue(0)                                                    # intra_chroma_pred_mode DC
                bw.se(0)                                                    # mb_qp_delta
                residual_block(bw, m['ldc'], left_tc[0] if c else 0)       # Intra16x16DCLevel: nC of block 0
            else:
                bw.ue(0)                                                    # mb_type P_L0_16x16
                bw.se(m['mv'][0] - mvp[0])
                bw.se(m['mv'][1] - mvp[1])
                mvp = m['mv']
                bw.ue(CBP_CODE[cbp_l + 16 * cbp_c])
                if cbp_l or cbp_c:
                    bw.se(0)                                                # mb_qp_delta
            for k, (bx, by) in enumerate(BLK):
                if cbp_l >> (k // 4) & 1:
                    na = tc[by, bx - 1] if bx else left_tc[by] if c else None
                    tc[by, bx] = residual_block(bw, m['lac'][k][1:] if idr else m['lac'][k], _nc(na, tc[by - 1, bx] if by else None))
            cc = [np.zeros((2, 2), int), np.zeros((2, 2), int)]
            if cbp_c:
                for comp in range(2):
                    residual_block(bw, m['cdc'][comp], -1)
            if cbp_c == 2:
                for comp in range(2):
                    for k in range(4):
                        by, bx = divmod(k, 2)
                        na = cc[comp][by, bx - 1] if bx else left_cc[comp][by] if c else None
                        cc[comp][by, bx] = residual_block(bw, m['cac'][comp][k][1:], _nc(na, cc[comp][by - 1, bx] if by else None))
            left_tc = [int(tc[by, 3]) for by in range(4)]
            left_cc = [[int(cc[comp][by, 1]) for by in range(2)] for comp in range(2)]
        if skip_run:
            bw.ue(skip_run)
        rbsp = bw.rbsp()
        nal = bytes([0x65 if idr else 0x61]) + escape(rbsp)
        if rec is not None:
            if skip_run:
                rec['skip run', 'whole row' if skip_run == len(mbs) else 'row end'] += 1
            rec['emulation prevention bytes'] += len(nal) - 1 - len(rbsp)
            rec['slice bytes max'] = max(rec['slice bytes max'], 4 + len(nal))
        return len(nal).to_bytes(4, 'big') + nal

    def encode(self, rgb):
        """One uint8 RGB frame [H, W, 3] -> (AVCC sample bytes, is_idr)."""
        rgb = np.asarray(rgb)
        if rgb.shape != (self.H, self.W, 3) or rgb.dtype != np.uint8:
            raise ValueError(f'expected a uint8 frame of shape {(self.H, self.W, 3)}, got {rgb.dtype} {rgb.shape}')
        Y, U, V = rgb_to_yuv420(rgb)
        k = self.n % self.gop
        idr = k == 0
        if idr:
            mbs, rec = self._intra(Y, U, V)
            self.mvs, self.skip, self.levels = None, None, None
        else:
            mbs, rec = self._inter(Y, U, V)
        R, C = self.mbh, self.mbw
        self.recon = tuple(p.swapaxes(1, 2).reshape(R * p.shape[2], C * p.shape[3]).astype(np.uint8) for p in rec)
        idr_pic_id = (self.n // self.gop) % 2
        if self.census is not None:
            self._record_frame(idr, k, idr_pic_id)
        sample = b''.join(self._slice(r, mbs[r], idr, k % 16, idr_pic_id) for r in range(R))
        self.n += 1
        return sample, idr


    def record(self, census):
        """Counts the syntax elements and decisions of the frames encoded from now on into census (a Counter; None stops).  The
        bytes do not change."""
        self.census = census
        return self

    def _record_frame(self, idr, k, idr_pic_id):
        rec, W, H, R, C = self.census, self.W, self.H, self.mbh, self.mbw
        rec['qp', 'I' if idr else 'P', self.qp] += 1
        rec['frame_num wrap',] += int(k > 0 and k % 16 == 0)
        if idr:
            rec['idr_pic_id', idr_pic_id] += 1
        for name, hit in (('2-sample crop remainder', W % 16 == 2 or H % 16 == 2), ('more than 32 MB rows', R > 32),
                          ('more than 256 MB rows', R > 256), ('1 MB column, several rows', C == 1 and R > 1),
                          ('2 MB columns, several rows', C == 2 and R > 1), ('more than 1024 MB columns', C > 1024)):
            rec['size', name] += int(hit)


def unblocks_dc(dc):
    """[..., 16] DC per luma4x4BlkIdx -> [..., 4, 4] spatial (row = block y, column = block x)."""
    out = np.zeros(dc.shape[:-1] + (4, 4), dc.dtype)
    for k, (bx, by) in enumerate(BLK):
        out[..., by, bx] = dc[..., k]
    return out


def blocks_dc(m):
    """Inverse of unblocks_dc."""
    return np.stack([m[..., by, bx] for bx, by in BLK], -1)


# ------------------------------------------------------------------------------------------------ quarter-sample luma
def _tap(p, axis):
    """6-tap filter (1, -5, 20, 20, -5, 1) between sample k and k + 1 along axis (unscaled; wraps at the borders, which PAD
    keeps out of use)."""
    s = lambda k: np.roll(p, -k, axis)
    return s(-2) - 5 * s(-1) + 20 * s(0) + 20 * s(1) - 5 * s(2) + s(3)


def half_planes(y):
    """Reference luma [H16, W16] -> (G, b, h, j) planes padded by PAD: full samples (edge replication = the decoder's clamped
    coordinates) and the half-sample positions right of, below, and right of and below each full sample."""
    G = np.pad(y.astype(np.int64), PAD, mode='edge')
    b1, h1 = _tap(G, 1), _tap(G, 0)
    clip = lambda v: np.clip(v, 0, 255)
    return G, clip((b1 + 16) >> 5), clip((h1 + 16) >> 5), clip((_tap(b1, 0) + 512) >> 10)


def luma_pred(P, X4, Y4):
    """Luma prediction samples at quarter-sample positions (X4, Y4) (arrays, picture coordinates * 4), Table 8-12."""
    G, B, Hh, J = P
    x, y = (X4 >> 2) + PAD, (Y4 >> 2) + PAD
    fx, fy = X4 & 3, Y4 & 3
    g, hh, m_, b, h, j, m, s = G[y, x], G[y, x + 1], G[y + 1, x], B[y, x], Hh[y, x], J[y, x], Hh[y, x + 1], B[y + 1, x]
    av = lambda a, c: (a + c + 1) >> 1
    table = [[g, av(g, b), b, av(hh, b)],
             [av(g, h), av(b, h), av(b, j), av(b, m)],
             [h, av(h, j), j, av(j, m)],
             [av(m_, h), av(h, s), av(j, s), av(m, s)]]
    out = np.zeros(np.broadcast(X4, Y4).shape, np.int64)
    for yf in range(4):
        for xf in range(4):
            sel = (fx == xf) & (fy == yf)
            out = np.where(sel, table[yf][xf], out)
    return out


# ------------------------------------------------------------------------------------------------ deblocking (8.7)
# Table 8-16 (alpha', beta') and Table 8-17 (tC0' for bS = 1, 2, 3), indexed by indexA / indexB
ALPHA = [0] * 16 + [4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25, 28, 32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113, 127,
                    144, 162, 182, 203, 226, 255, 255]
BETA = [0] * 16 + [2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16, 17,
                   17, 18, 18]
TC0 = [(0, 0, 0)] * 17 + [(0, 0, 1)] * 4 + [(0, 1, 1)] * 2 + [(1, 1, 1)] * 4 + [(1, 1, 2)] * 4 + [(1, 2, 3)] * 2 + [
    (2, 2, 3), (2, 2, 4), (2, 3, 4), (2, 3, 4), (3, 3, 5), (3, 4, 6), (3, 4, 6), (4, 5, 7), (4, 5, 8), (4, 6, 9), (5, 7, 10),
    (6, 8, 11), (6, 8, 13), (7, 10, 14), (8, 11, 16), (9, 12, 18), (10, 13, 20), (11, 15, 23), (13, 17, 25)]


def _filter(s, bS, idx, chroma, census=None):
    """Filter lines across one edge: s [..., 8] luma samples p3..q3, or [..., 4] chroma p1..q1; bS [...]; idx = indexA = indexB.
    census (a Counter, or None) counts the lines per (bS, whether the sample test |p0 - q0| < alpha, |p1 - p0| < beta,
    |q1 - q0| < beta passes), so that bS 0 with a passing test (no filtering all the same) is counted too."""
    a, be = ALPHA[idx], BETA[idx]
    if chroma:
        p1, p0, q0, q1 = (s[..., k] for k in range(4))
    else:
        p3, p2, p1, p0, q0, q1, q2, q3 = (s[..., k] for k in range(8))
    test = (np.abs(p0 - q0) < a) & (np.abs(p1 - p0) < be) & (np.abs(q1 - q0) < be)
    on = (bS > 0) & test
    if census is not None:
        for b in range(5):
            for t in (True, False):
                census['bS', 'chroma' if chroma else 'luma', b, 'filtered' if t else 'not filtered'] += int(((bS == b) & (test == t)).sum())
    weak, strong = on & (bS < 4), on & (bS == 4)
    tc0 = np.array((0,) + TC0[idx])[np.minimum(bS, 3)]
    out = s.copy()
    if chroma:
        tc = tc0 + 1
    else:
        ap, aq = np.abs(p2 - p0) < be, np.abs(q2 - q0) < be
        tc = tc0 + ap + aq
    delta = np.clip((((q0 - p0) << 2) + (p1 - q1) + 4) >> 3, -tc, tc)
    w_p0, w_q0 = np.clip(p0 + delta, 0, 255), np.clip(q0 - delta, 0, 255)
    if chroma:
        out[..., 1] = np.where(weak, w_p0, np.where(strong, (2 * p1 + p0 + q1 + 2) >> 2, p0))
        out[..., 2] = np.where(weak, w_q0, np.where(strong, (2 * q1 + q0 + p1 + 2) >> 2, q0))
        return out
    w_p1 = np.where(ap, p1 + np.clip((p2 + ((p0 + q0 + 1) >> 1) - (p1 << 1)) >> 1, -tc0, tc0), p1)
    w_q1 = np.where(aq, q1 + np.clip((q2 + ((p0 + q0 + 1) >> 1) - (q1 << 1)) >> 1, -tc0, tc0), q1)
    near = np.abs(p0 - q0) < ((a >> 2) + 2)
    sp, sq = ap & near, aq & near
    s_p0 = np.where(sp, (p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3, (2 * p1 + p0 + q1 + 2) >> 2)
    s_p1 = np.where(sp, (p2 + p1 + p0 + q0 + 2) >> 2, p1)
    s_p2 = np.where(sp, (2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3, p2)
    s_q0 = np.where(sq, (p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3, (2 * q1 + q0 + p1 + 2) >> 2)
    s_q1 = np.where(sq, (p0 + q0 + q1 + q2 + 2) >> 2, q1)
    s_q2 = np.where(sq, (2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3, q2)
    for k, wv, sv in ((1, p2, s_p2), (2, w_p1, s_p1), (3, w_p0, s_p0), (4, w_q0, s_q0), (5, w_q1, s_q1), (6, q2, s_q2)):
        out[..., k] = np.where(weak, wv, np.where(strong, sv, s[..., k]))
    return out


def boundary_strength(intra, nz, mv):
    """bS of the vertical (left, then internal) and horizontal (top, then internal) luma edges of every MB: [R, C, edge, 4]
    (index along the edge in 4x4 blocks).  intra: the picture is intra; nz [R, C, 4, 4] (by, bx): the luma 4x4 block has
    nonzero levels; mv [R, C, 2] quarter samples.  Picture borders get 0."""
    R, C = nz.shape[:2]
    bv, bh = np.zeros((R, C, 4, 4), np.int64), np.zeros((R, C, 4, 4), np.int64)
    if intra:
        bv[:, :, 1:], bh[:, :, 1:] = 3, 3
        bv[:, 1:, 0], bh[1:, :, 0] = 4, 4
        return bv, bh
    for e in range(1, 4):
        bv[:, :, e] = 2 * (nz[:, :, :, e - 1] | nz[:, :, :, e])
        bh[:, :, e] = 2 * (nz[:, :, e - 1, :] | nz[:, :, e, :])
    mvd = lambda a, c: (np.abs(a - c) >= 4).any(-1)[..., None]
    bv[:, 1:, 0] = np.where(nz[:, 1:, :, 0] | nz[:, :-1, :, 3], 2, mvd(mv[:, 1:], mv[:, :-1]))
    bh[1:, :, 0] = np.where(nz[1:, :, 0, :] | nz[:-1, :, 3, :], 2, mvd(mv[1:], mv[:-1]))
    return bv, bh


def deblock(planes, qp, bv, bh, census=None):
    """In-place deblocking of padded (Y, Cb, Cr) int64 planes in the standard's order (per MB in raster order: vertical edges
    left to right, then horizontal edges top to bottom), run on the MBs of one wavefront x + 2y at a time: an MB's filtering only
    touches samples that the MBs to its left and above-right finished with."""
    Y, U, V = planes
    R, C = bv.shape[:2]
    qpc = QPC[qp]
    ar = np.arange
    for t in range(C + 2 * (R - 1)):
        r = ar(R)[(t - 2 * ar(R) >= 0) & (t - 2 * ar(R) < C)]
        c = t - 2 * r
        for vertical in (True, False):
            bs = bv if vertical else bh
            for e in range(4):
                sel = (c > 0) if (vertical and e == 0) else (r > 0) if e == 0 else np.ones(len(r), bool)
                rr, cc = r[sel], c[sel]
                if not len(rr):
                    continue
                strength = bs[rr, cc, e]                                                 # [n, 4]
                along = lambda base, n, k: base[:, None] + ar(n)[None, :] + k
                if vertical:                                                             # lines = rows, samples across columns
                    iy, ix = along(16 * rr, 16, 0)[:, :, None], along(16 * cc + 4 * e, 8, -4)[:, None, :]
                else:
                    iy, ix = along(16 * rr + 4 * e, 8, -4)[:, None, :], along(16 * cc, 16, 0)[:, :, None]
                Y[iy, ix] = _filter(Y[iy, ix], np.repeat(strength, 4, 1), qp, False, census)
                if e % 2:
                    continue
                cs = np.repeat(strength, 2, 1)                                            # chroma edge 4e/2 = luma edge e
                if vertical:
                    iy, ix = along(8 * rr, 8, 0)[:, :, None], along(8 * cc + 2 * e, 4, -2)[:, None, :]
                else:
                    iy, ix = along(8 * rr + 2 * e, 4, -2)[:, None, :], along(8 * cc, 8, 0)[:, :, None]
                for p in (U, V):
                    p[iy, ix] = _filter(p[iy, ix], cs, qpc, True, census)


# ------------------------------------------------------------------------------------------------ rate control
def _fdiv(a, b):
    return a // b                                     # floor division (b > 0); the device states it explicitly


class RateControl:
    """The device controller (csrc/h264.cu h264_rc_update), in the same integer arithmetic.  A leaky bucket of one second: fullness
    is the stream's excess over bitrate x time, in 1/fps_num bits, saturating at +-8 s.  The budget of the next frame is the per-frame rate minus a
    second's share of the fullness; after each P frame (and after an IDR frame that follows an IDR frame) QP moves by -2..+2 by
    how far that frame's bits were from its budget.  IDR frames keep the QP of the P frames around them and are paid for by the
    P frames after them."""

    def __init__(self, width, height, bitrate, fps_num, fps_den, qp_min=0, qp_max=51):
        self.bitrate, self.num, self.den, self.qp_min, self.qp_max = bitrate, fps_num, fps_den, qp_min, qp_max
        self.fullness, self.frames, self.prev_idr = 0, 0, 0
        x, y, q = 10 * bitrate * fps_den, fps_num * width * height, 30              # 30 at 0.1 bits per pixel, -6 per doubling
        while x >= 2 * y and q > 0:
            y, q = 2 * y, q - 6
        while 2 * x < y and q < 51:
            x, q = 2 * x, q + 6
        self.qp = min(max(q, qp_min), qp_max)

    def update(self, nbytes, idr, census=None):
        """census (a Counter, or None) counts the steps, the clamps at the QP bounds and the updates after an IDR frame that
        follows an IDR frame."""
        bits = 8 * nbytes * self.num
        budget = self.bitrate * self.den
        sat = 8 * self.bitrate * self.num                        # the bucket saturates at +-8 s
        self.fullness = min(max(self.fullness + bits - budget, -sat), sat)
        if not idr or self.prev_idr:
            want = max(budget - _fdiv(self.fullness, max(1, self.num // self.den)), budget // 8)
            step = (2 if 100 * bits > 141 * want else 1 if 100 * bits > 112 * want else
                    -2 if 141 * bits < 100 * want else -1 if 112 * bits < 100 * want else 0)
            if census is not None:
                census['rc', f'step {step:+d}'] += 1
                census['rc', 'clamped at qp_min'] += int(self.qp + step < self.qp_min)
                census['rc', 'clamped at qp_max'] += int(self.qp + step > self.qp_max)
                census['rc', 'IDR frame after an IDR frame'] += int(idr)
            self.qp = min(max(self.qp + step, self.qp_min), self.qp_max)
        self.prev_idr = int(idr)
        self.frames += 1


# ------------------------------------------------------------------------------------------------ rate-controlled stream
class RcEncoder(Encoder):
    """The rate-controlled stream: Encoder's coding with a controller-chosen QP per picture, quarter-sample motion and deblocking.
    bitrate in bits/s, fps = (num, den); qp_min == qp_max pins the QP.  After each encode(): recon is the deblocked picture, qps
    the QP of every frame so far."""

    def __init__(self, width, height, bitrate, fps=(30, 1), gop=60, qp_min=0, qp_max=51):
        super().__init__(width, height, 26, gop)
        self.rc = RateControl(width, height, bitrate, fps[0], fps[1], qp_min, qp_max)
        self.qps = []

    def _search(self, ry, cur):
        """The integer search, then the 8 half-sample neighbours of its vector, then the 8 quarter-sample neighbours of the best of
        those, with the same cost and key; luma predicted with the 6-tap filter (8.4.2.2.1)."""
        P = half_planes(ry)
        best = self._integer_search(P[0], cur)
        qx, qy = mv_of(best)
        src = _mb_view(cur, 16)
        lam = LAMBDA[self.qp]
        X0 = 4 * (16 * np.arange(self.mbw)[None, :, None, None] + np.arange(16)[None, None, None, :])
        Y0 = 4 * (16 * np.arange(self.mbh)[:, None, None, None] + np.arange(16)[None, None, :, None])
        pred_at = lambda x, y: luma_pred(P, X0 + x[:, :, None, None], Y0 + y[:, :, None, None])
        for step in (2, 1):
            cx, cy = qx, qy
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    if dx or dy:
                        x, y = cx + step * dx, cy + step * dy
                        cost = np.abs(src - pred_at(x, y)).sum((-1, -2)) + lam * (se_bits(x) + se_bits(y))
                        np.minimum(best, mv_key(cost, x, y), out=best)
            qx, qy = mv_of(best)
        return qx, qy, pred_at(qx, qy)

    def _slice_qp_and_deblocking(self, bw):
        bw.se(self.qp - 26)                        # slice_qp_delta (pic_init_qp 26)
        bw.ue(0)                                   # disable_deblocking_filter_idc: filter, across slice boundaries too
        bw.se(0)                                   # slice_alpha_c0_offset_div2
        bw.se(0)                                   # slice_beta_offset_div2

    def encode(self, rgb):
        """Codes the frame at the controller's QP, then deblocks the reconstruction (the slices do not depend on it) and updates
        the controller with the sample's size."""
        self.qp = self.rc.qp
        sample, idr = super().encode(rgb)
        R, C = self.mbh, self.mbw
        if idr:
            nz, mv = np.zeros((R, C, 4, 4), bool), np.zeros((R, C, 2), np.int64)
        else:
            nz, mv = unblocks_dc(self.levels.any((-1, -2))), self.mvs
        planes = tuple(p.astype(np.int64) for p in self.recon)
        deblock(planes, self.qp, *boundary_strength(idr, nz, mv), self.census)
        self.recon = tuple(p.astype(np.uint8) for p in planes)
        self.rc.update(len(sample), idr, self.census)
        self.qps.append(self.qp)
        return sample, idr


# ------------------------------------------------------------------------------------------------ test sequences
TRANSLATE = (3, -1)             # per-frame shift of the 'translate' sequence: frame t samples the pattern at x + 3t, y - t
EDGE = (2, 2)                   # ... and of 'edge', whose pattern has a hard border that moves across the picture


def _pattern(H, W, seed):
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    img = np.zeros((H, W, 3))
    for c in range(3):
        for _ in range(6):
            fx, fy, ph = rng.uniform(0.02, 0.25, 2).tolist() + [rng.uniform(0, 6.3)]
            img[..., c] += np.sin(fx * x + fy * y + ph) * rng.uniform(10, 30)
    return np.clip(img + 128, 0, 255).astype(np.uint8)


def sequence(name, W, H, n=3):
    """n uint8 RGB frames [H, W, 3] of one of the named test sequences."""
    if name == 'flat':
        return [np.full((H, W, 3), (40 + 60 * t, 120, 200 - 50 * t), np.uint8) for t in range(n)]
    if name == 'gradient':
        y, x = np.mgrid[0:H, 0:W]
        return [np.stack([(x * 255 // max(W - 1, 1) + 4 * t) % 256, y * 255 // max(H - 1, 1), np.full_like(x, 90 + 10 * t)],
                         -1).astype(np.uint8) for t in range(n)]
    if name in ('translate', 'edge'):
        dx, dy = TRANSLATE if name == 'translate' else EDGE
        m = 4 * n + 8
        big = _pattern(H + 2 * m, W + 2 * m, 1)
        if name == 'edge':                                   # a flat region whose border moves into the picture
            big[:, :m + W // 2] = (30, 200, 60)
        return [big[m + dy * t:m + dy * t + H, m + dx * t:m + dx * t + W].copy() for t in range(n)]
    if name == 'noise':
        rng = np.random.RandomState(W * 1000 + H)
        return [rng.randint(0, 256, (H, W, 3)).astype(np.uint8) for _ in range(n)]
    raise ValueError(name)


SEQUENCES = ('flat', 'gradient', 'translate', 'edge', 'noise')

PAN = (1.25, -0.5)              # per-frame shift of the 'pan' sequence: frame t samples the pattern at x + 1.25t, y - 0.5t
PAN_SCALE = 3                   # ... with _pattern's frequencies times 3 (at most 0.75 rad/sample per term), so that a quarter
                                # sample of motion moves the SAD well above the reconstruction's noise at QP 18


def pan(W, H, n=3):
    """n uint8 RGB frames [H, W, 3] of _pattern's analytic pattern (frequencies scaled by PAN_SCALE) panned by a fraction of a
    sample per frame (true vector (5, -2) in quarter samples)."""
    out = []
    for t in range(n):
        rng = np.random.RandomState(1)
        y, x = np.mgrid[0:H, 0:W].astype(np.float64)
        x, y = PAN_SCALE * (x + PAN[0] * t), PAN_SCALE * (y + PAN[1] * t)
        img = np.zeros((H, W, 3))
        for c in range(3):
            for _ in range(6):
                fx, fy, ph = rng.uniform(0.02, 0.25, 2).tolist() + [rng.uniform(0, 6.3)]
                img[..., c] += np.sin(fx * x + fy * y + ph) * rng.uniform(10, 30)
        out.append(np.clip(img + 128, 0, 255).astype(np.uint8))
    return out


# ------------------------------------------------------------------------------------------------ edge sequences
# Built to reach the coding edges the sequences above do not (tests/test_h264_edges_cpu.py counts what they reach):
# - 'stripes': 16-sample blue / yellow columns under noise, the colours swapping every frame.  At QP 0 the I_16x16 luma DC and the
#   chroma DC of every MB after the first column exceed LEVEL_MAX, the noise fills every AC coefficient with large levels (escape
#   codes, suffixLength 6), and the P frames match the swapped columns at +-16 samples, the search bound.
# - 'cut': flat yellow, flat blue, then noise: a P frame whose chroma DC exceeds LEVEL_MAX, then a scene cut inside the GOP (a P
#   frame with IDR-sized residuals).
# - 'static': a still picture in which a sparse set of MBs shows the picture zoomed about its centre (a little more every
#   frame): skip runs at the start, in the middle and at the end of a row, rows of skips, and a vector field that takes every
#   quarter-sample position.
# - 'motion': the smooth pattern moved by (+16.75, -16.75), (-16.75, +16.75), then (+24, +24) samples per frame: vectors at the
#   search bound refined past it, and motion beyond it, with the reference blocks of the border MBs wholly outside the frame.
# - 'cbp': a still, softened pattern; in the P frames MB k gets grey noise in the 8x8 quadrants of the bits of k % 16 and, by
#   (k // 16 + t - 1) % 3 in frame t, no change of colour, a flat tint (chroma DC only) or a tint in a checker of 4x4 blocks (chroma AC): at
#   moderate QPs, with 48 MBs, every coded_block_pattern of a P MB.
# - 'mosaic': MB-sized tiles (flat grey, grey noise, a flat colour, grey noise, the rows of the left tile's last column tinted,
#   the smooth pattern) that make every I_16x16 mb_type across the QPs; the noise and the pattern change in every frame.
EDGE_SEQUENCES = ('stripes', 'cut', 'static', 'motion', 'cbp', 'mosaic')
TINT = (39, -20, 0)                                 # an RGB offset that moves Cb and Cr but not Y (66 * 39 - 129 * 20 = -6)
BLUE, YELLOW = (0, 0, 255), (255, 255, 0)           # Y 41 / 210, Cb 240 / 16: far apart in luma and in Cb
MOTION = [(16.75, -16.75), (-16.75, 16.75), (24, 24)]


def _smooth(H, W, ox=0.0, oy=0.0, zoom=1.0):
    """_pattern's analytic pattern sampled at ((x - W/2) / zoom + W/2 + ox, (y - H/2) / zoom + H/2 + oy)."""
    rng = np.random.RandomState(1)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    x, y = (x - W / 2) / zoom + W / 2 + ox, (y - H / 2) / zoom + H / 2 + oy
    img = np.zeros((H, W, 3))
    for c in range(3):
        for _ in range(6):
            fx, fy, ph = rng.uniform(0.02, 0.25, 2).tolist() + [rng.uniform(0, 6.3)]
            img[..., c] += np.sin(fx * x + fy * y + ph) * rng.uniform(10, 30)
    return np.clip(img + 128, 0, 255).astype(np.uint8)


def edge_sequence(name, W, H, n=3):
    """n uint8 RGB frames [H, W, 3] of one of EDGE_SEQUENCES."""
    if name == 'stripes':
        col = (np.arange(W) // 16) % 2
        out = []
        for t in range(n):
            base = np.where((col ^ (t % 2))[None, :, None] == 1, BLUE, YELLOW) * np.ones((H, 1, 1), np.int64)
            noise = np.random.RandomState(7 + t).randint(-48, 49, (H, W, 3))
            out.append(np.clip(base + noise, 0, 255).astype(np.uint8))
        return out
    if name == 'cut':
        pics = [lambda: np.full((H, W, 3), YELLOW, np.uint8), lambda: np.full((H, W, 3), BLUE, np.uint8),
                lambda: np.random.RandomState(11).randint(0, 256, (H, W, 3)).astype(np.uint8)]
        return [pics[t % 3]() for t in range(n)]
    if name == 'static':
        still = _smooth(H, W)
        R, C = (H + 15) // 16, (W + 15) // 16
        out = [still]
        for t in range(1, n):
            zoomed = _smooth(H, W, zoom=1 + 0.02 * t)
            f = still.copy()
            for r in range(0, R, 3):                       # rows 0, 3, 6, ...: MB columns 1, 6, 11, ... (column 0 if it is the only one)
                for c in range(min(1, C - 1), C, 5):
                    f[16 * r:16 * r + 16, 16 * c:16 * c + 16] = zoomed[16 * r:16 * r + 16, 16 * c:16 * c + 16]
            out.append(f)
        return out
    if name == 'cbp':
        still = (_smooth(H, W).astype(np.int64) - 128) // 3 + 128
        R, C = (H + 15) // 16, (W + 15) // 16
        out = [still.astype(np.uint8)]
        for t in range(1, n):
            rng = np.random.RandomState(20 + t)
            f = still.copy()
            for k in range(R * C):
                y0, x0 = 16 * (k // C), 16 * (k % C)
                for q in range(4):
                    if k % 16 >> q & 1:
                        ys, xs = slice(y0 + 8 * (q // 2), y0 + 8 * (q // 2) + 8), slice(x0 + 8 * (q % 2), x0 + 8 * (q % 2) + 8)
                        f[ys, xs] += rng.randint(-24, 25, f[ys, xs].shape[:2])[..., None]
                tint = (k // 16 + t - 1) % 3
                if tint:
                    sign = np.ones((16, 16), np.int64) if tint == 1 else np.kron([[1, -1, 1, -1], [-1, 1, -1, 1]] * 2, np.ones((4, 4), np.int64))
                    f[y0:y0 + 16, x0:x0 + 16] += (sign[..., None] * TINT)[:f[y0:y0 + 16].shape[0], :f[:, x0:x0 + 16].shape[1]]
            out.append(np.clip(f, 0, 255).astype(np.uint8))
        return out
    if name == 'mosaic':
        R, C = (H + 15) // 16, (W + 15) // 16
        out = []
        for t in range(n):
            rng = np.random.RandomState(30 + t)
            f = np.zeros((16 * R, 16 * C, 3), np.int64)
            smooth = _smooth(16 * R, 16 * C, 1.25 * t, -0.5 * t)
            for k in range(R * C):
                y0, x0 = 16 * (k // C), 16 * (k % C)
                tile = f[y0:y0 + 16, x0:x0 + 16]
                kind = k % 6
                if kind == 0:
                    tile[:] = 128
                elif kind in (1, 3):
                    tile[:] = rng.randint(40, 200, (16, 16))[..., None]
                elif kind == 2:
                    tile[:] = (200, 120, 60)
                elif kind == 4:
                    left = f[y0:y0 + 16, x0 - 1] if x0 else np.full((16, 3), 128)
                    tile[:] = (left + TINT)[:, None, :]
                else:
                    tile[:] = smooth[y0:y0 + 16, x0:x0 + 16]
            out.append(np.clip(f[:H, :W], 0, 255).astype(np.uint8))
        return out
    if name == 'motion':
        o, out = np.zeros(2), []
        for t in range(n):
            out.append(_smooth(H, W, *o))
            o = o + MOTION[t % len(MOTION)]
        return out
    raise ValueError(name)


def frames(name, W, H, n=3):
    """sequence(), 'pan' and edge_sequence()."""
    if name == 'pan':
        return pan(W, H, n)
    return edge_sequence(name, W, H, n) if name in EDGE_SEQUENCES else sequence(name, W, H, n)
