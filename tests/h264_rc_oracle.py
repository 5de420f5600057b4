"""numpy restatement of the rate-controlled H.264 stream of csrc/h264.cu (n3d_h264_encode_rc): quarter-sample motion
(8.4.2.2.1), the in-loop deblocking filter (8.7) in the standard's order, and the device's integer rate controller.  It builds on
tests/h264_oracle.py, whose constant-QP `Encoder` it leaves unchanged: `RcEncoder` reuses its colour conversion, intra coding,
transforms and CAVLC, and makes the same decisions as the kernels, so the GPU tests compare bytes and reconstructions exactly.

Stream differences from the constant-QP one: pic_init_qp 26 with slice_qp_delta = QP - 26 (one QP per picture, chosen by the
controller before the picture is coded), P_L0_16x16 vectors refined to quarter samples around the integer search's best vector,
and disable_deblocking_filter_idc 0 (the deblocked picture is the output and the next P frame's reference)."""
import numpy as np

from tests import h264_oracle as O

# Table 8-16 (alpha', beta') and Table 8-17 (tC0' for bS = 1, 2, 3), indexed by indexA / indexB
ALPHA = [0] * 16 + [4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25, 28, 32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113, 127,
                    144, 162, 182, 203, 226, 255, 255]
BETA = [0] * 16 + [2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16, 17,
                   17, 18, 18]
TC0 = [(0, 0, 0)] * 17 + [(0, 0, 1)] * 4 + [(0, 1, 1)] * 2 + [(1, 1, 1)] * 4 + [(1, 1, 2)] * 4 + [(1, 2, 3)] * 2 + [
    (2, 2, 3), (2, 2, 4), (2, 3, 4), (2, 3, 4), (3, 3, 5), (3, 4, 6), (3, 4, 6), (4, 5, 7), (4, 5, 8), (4, 6, 9), (5, 7, 10),
    (6, 8, 11), (6, 8, 13), (7, 10, 14), (8, 11, 16), (9, 12, 18), (10, 13, 20), (11, 15, 23), (13, 17, 25)]
PAD = O.SEARCH + 8              # reference padding: covers the search, the quarter-sample refinement and the 6-tap filter
MV_OFF = 128                    # key offset of quarter-sample vector components (|mv| <= 4 * SEARCH + 3)
RC_FIELDS = 16                  # int64 fields of the controller state (N3D_H264_RC_STATE_BYTES / 8)


def _bits(k):
    """ue(v) length of code numbers k (array)."""
    return 2 * np.frexp(np.asarray(k, np.float64) + 1)[1].astype(np.int64) - 1


def _se(v):
    v = np.asarray(v, np.int64)
    return np.where(v > 0, 2 * v - 1, -2 * v)


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
def _filter(s, bS, idx, chroma):
    """Filter lines across one edge: s [..., 8] luma samples p3..q3, or [..., 4] chroma p1..q1; bS [...]; idx = indexA = indexB."""
    a, be = ALPHA[idx], BETA[idx]
    if chroma:
        p1, p0, q0, q1 = (s[..., k] for k in range(4))
    else:
        p3, p2, p1, p0, q0, q1, q2, q3 = (s[..., k] for k in range(8))
    on = (bS > 0) & (np.abs(p0 - q0) < a) & (np.abs(p1 - p0) < be) & (np.abs(q1 - q0) < be)
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


def deblock(planes, qp, bv, bh):
    """In-place deblocking of padded (Y, Cb, Cr) int64 planes in the standard's order (per MB in raster order: vertical edges
    left to right, then horizontal edges top to bottom), run on the MBs of one wavefront x + 2y at a time: an MB's filtering only
    touches samples that the MBs to its left and above-right finished with."""
    Y, U, V = planes
    R, C = bv.shape[:2]
    qpc = O.QPC[qp]
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
                Y[iy, ix] = _filter(Y[iy, ix], np.repeat(strength, 4, 1), qp, False)
                if e % 2:
                    continue
                cs = np.repeat(strength, 2, 1)                                            # chroma edge 4e/2 = luma edge e
                if vertical:
                    iy, ix = along(8 * rr, 8, 0)[:, :, None], along(8 * cc + 2 * e, 4, -2)[:, None, :]
                else:
                    iy, ix = along(8 * rr + 2 * e, 4, -2)[:, None, :], along(8 * cc, 8, 0)[:, :, None]
                for p in (U, V):
                    p[iy, ix] = _filter(p[iy, ix], cs, qpc, True)


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

    def update(self, nbytes, idr):
        bits = 8 * nbytes * self.num
        budget = self.bitrate * self.den
        sat = 8 * self.bitrate * self.num                        # the bucket saturates at +-8 s
        self.fullness = min(max(self.fullness + bits - budget, -sat), sat)
        if not idr or self.prev_idr:
            want = max(budget - _fdiv(self.fullness, max(1, self.num // self.den)), budget // 8)
            step = (2 if 100 * bits > 141 * want else 1 if 100 * bits > 112 * want else
                    -2 if 141 * bits < 100 * want else -1 if 112 * bits < 100 * want else 0)
            self.qp = min(max(self.qp + step, self.qp_min), self.qp_max)
        self.prev_idr = int(idr)
        self.frames += 1


# ------------------------------------------------------------------------------------------------ encoder
class RcEncoder(O.Encoder):
    """The rate-controlled stream: O.Encoder's intra coding and syntax with a controller-chosen QP per picture, quarter-sample
    motion and deblocking.  bitrate in bits/s, fps = (num, den); qp_min == qp_max pins the QP.  After each encode(): recon is
    the deblocked picture, mvs [mbh, mbw, 2] the P frame's vectors in quarter samples, qps the QP of every frame so far."""

    def __init__(self, width, height, bitrate, fps=(30, 1), gop=60, qp_min=0, qp_max=51):
        super().__init__(width, height, 26, gop)
        self.rc = RateControl(width, height, bitrate, fps[0], fps[1], qp_min, qp_max)
        self.qps = []

    def _inter(self, Y, U, V):
        qp, qpc = self.qp, O.QPC[self.qp]
        R, C = self.mbh, self.mbw
        H16, W16 = 16 * R, 16 * C
        ry, ru, rv = (p.astype(np.int64) for p in self.recon)
        cur = Y.astype(np.int64)
        src = O._mb_view(cur, 16)
        P = half_planes(ry)
        lam = O.LAMBDA[qp]
        S = O.SEARCH
        best = np.full((R, C), np.iinfo(np.int64).max, np.int64)
        mx = np.arange(-S, S + 1)
        for my in range(-S, S + 1):                   # integer-pel full search, as the constant-QP encoder (all mx at once)
            rows = P[0][PAD + my:PAD + my + H16, PAD - S:PAD + S + W16]
            shifted = np.lib.stride_tricks.sliding_window_view(rows, W16, 1).swapaxes(0, 1)              # [mx, H16, W16]
            sad = np.abs(cur - shifted).reshape(2 * S + 1, R, 16, C, 16).sum((2, 4))
            cost = sad + lam * (_bits(_se(4 * mx)) + O.ue_bits(O.se_code(4 * my)))[:, None, None]
            keys = (cost << 24) | ((np.abs(mx) + abs(my)) << 16)[:, None, None] | ((my + S) << 8) | (mx + S)[:, None, None]
            np.minimum(best, keys.min(0), out=best)
        qx, qy = 4 * ((best & 0xff) - S), 4 * (((best >> 8) & 0xff) - S)
        X0 = 4 * (16 * np.arange(C)[None, :, None, None] + np.arange(16)[None, None, None, :])
        Y0 = 4 * (16 * np.arange(R)[:, None, None, None] + np.arange(16)[None, None, :, None])
        key = lambda cost, x, y: (cost << 24) | ((np.abs(x) + np.abs(y)) << 16) | ((y + MV_OFF) << 8) | (x + MV_OFF)
        best = key(best >> 24, qx, qy)
        for step in (2, 1):                           # the 8 half-sample neighbours, then the 8 quarter-sample ones of the best
            cx, cy = qx, qy
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    if dx or dy:
                        x, y = cx + step * dx, cy + step * dy
                        pred = luma_pred(P, X0 + x[:, :, None, None], Y0 + y[:, :, None, None])
                        cost = np.abs(src - pred).sum((-1, -2)) + lam * (_bits(_se(x)) + _bits(_se(y)))
                        np.minimum(best, key(cost, x, y), out=best)
            qx, qy = (best & 0xff) - MV_OFF, ((best >> 8) & 0xff) - MV_OFF
        pred = luma_pred(P, X0 + qx[:, :, None, None], Y0 + qy[:, :, None, None])
        w = O.fwd4(O.blocks(src - pred))
        lvl = O.quant(w, qp, False)
        rec_y = np.clip(pred + O.unblocks(O.inv4(O.dequant(lvl, qp))), 0, 255)
        fx, fy = (qx & 7)[:, :, None, None], (qy & 7)[:, :, None, None]             # chroma: eighth samples = luma quarters
        cy = np.arange(8)[None, None, :, None] + 8 * np.arange(R)[:, None, None, None] + (qy >> 3)[:, :, None, None]
        cx = np.arange(8)[None, None, None, :] + 8 * np.arange(C)[None, :, None, None] + (qx >> 3)[:, :, None, None]
        cres, crec = [], []
        for sp, rp in ((U, ru), (V, rv)):
            at = lambda yy, xx: rp[np.clip(yy, 0, H16 // 2 - 1), np.clip(xx, 0, W16 // 2 - 1)]
            cp = ((8 - fx) * (8 - fy) * at(cy, cx) + fx * (8 - fy) * at(cy, cx + 1) + (8 - fx) * fy * at(cy + 1, cx)
                  + fx * fy * at(cy + 1, cx + 1) + 32) >> 6
            dcl_c, acl_c, rec_c = O.code_chroma(O._mb_view(sp.astype(np.int64), 8), cp, qpc, False)
            cres.append((dcl_c, acl_c))
            crec.append(rec_c)
        nonzero = (lvl != 0).any((-1, -2, -3)) | (cres[0][0] != 0).any(-1) | (cres[0][1] != 0).any((-1, -2)) \
            | (cres[1][0] != 0).any(-1) | (cres[1][1] != 0).any((-1, -2))
        skip = (qx == 0) & (qy == 0) & ~nonzero
        mbs = [[dict(intra=False, skip=bool(skip[r, c]), mv=(int(qx[r, c]), int(qy[r, c])), lac=O.scan(lvl[r, c]),
                     cdc=[cres[0][0][r, c], cres[1][0][r, c]], cac=[cres[0][1][r, c], cres[1][1][r, c]])
                for c in range(C)] for r in range(R)]
        self.mvs, self.skip = np.stack([qx, qy], -1), skip
        return mbs, (rec_y, crec[0], crec[1])

    def _slice(self, row, mbs, idr, frame_num, idr_pic_id):
        """O.Encoder._slice with this stream's header fields (slice_qp_delta, deblocking on) and quarter-sample vectors."""
        bw = O.Bits()
        bw.ue(row * self.mbw)
        bw.ue(2 if idr else 0)
        bw.ue(0)
        bw.u(frame_num, 4)
        if idr:
            bw.ue(idr_pic_id)
        else:
            bw.u(0, 1)
            bw.u(0, 1)
        bw.u(0, 1)
        if idr:
            bw.u(0, 1)
        bw.se(self.qp - 26)                        # slice_qp_delta (pic_init_qp 26)
        bw.ue(0)                                   # disable_deblocking_filter_idc: filter, across slice boundaries too
        bw.se(0)                                   # slice_alpha_c0_offset_div2
        bw.se(0)                                   # slice_beta_offset_div2
        left_tc, left_cc, skip_run, mvp = [0] * 4, [[0, 0], [0, 0]], 0, (0, 0)
        for c, m in enumerate(mbs):
            if not idr and m['skip']:
                skip_run += 1
                left_tc, left_cc, mvp = [0] * 4, [[0, 0], [0, 0]], (0, 0)
                continue
            tc = np.zeros((4, 4), int)
            if idr:
                cbp_l = 15 if any(np.any(m['lac'][k][1:]) for k in range(16)) else 0
            else:
                bw.ue(skip_run)
                skip_run = 0
                cbp_l = sum(1 << q for q in range(4) if any(np.any(m['lac'][4 * q + k]) for k in range(4)))
            cbp_c = 2 if any(np.any(x[:, 1:]) for x in m['cac']) else 1 if any(np.any(x) for x in m['cdc']) else 0
            if idr:
                bw.ue(1 + m['mode'] + 4 * cbp_c + (12 if cbp_l else 0))
                bw.ue(0)
                bw.se(0)
                O.residual_block(bw, m['ldc'], left_tc[0] if c else 0)
            else:
                bw.ue(0)
                bw.se(m['mv'][0] - mvp[0])
                bw.se(m['mv'][1] - mvp[1])
                mvp = m['mv']
                bw.ue(O.CBP_CODE[cbp_l + 16 * cbp_c])
                if cbp_l or cbp_c:
                    bw.se(0)
            for k, (bx, by) in enumerate(O.BLK):
                if cbp_l >> (k // 4) & 1:
                    na = tc[by, bx - 1] if bx else left_tc[by] if c else None
                    tc[by, bx] = O.residual_block(bw, m['lac'][k][1:] if idr else m['lac'][k], O._nc(na, tc[by - 1, bx] if by else None))
            cc = [np.zeros((2, 2), int), np.zeros((2, 2), int)]
            if cbp_c:
                for comp in range(2):
                    O.residual_block(bw, m['cdc'][comp], -1)
            if cbp_c == 2:
                for comp in range(2):
                    for k in range(4):
                        by, bx = divmod(k, 2)
                        na = cc[comp][by, bx - 1] if bx else left_cc[comp][by] if c else None
                        cc[comp][by, bx] = O.residual_block(bw, m['cac'][comp][k][1:], O._nc(na, cc[comp][by - 1, bx] if by else None))
            left_tc = [int(tc[by, 3]) for by in range(4)]
            left_cc = [[int(cc[comp][by, 1]) for by in range(2)] for comp in range(2)]
        if skip_run:
            bw.ue(skip_run)
        nal = bytes([0x65 if idr else 0x61]) + O.escape(bw.rbsp())
        return len(nal).to_bytes(4, 'big') + nal

    def encode(self, rgb):
        rgb = np.asarray(rgb)
        if rgb.shape != (self.H, self.W, 3) or rgb.dtype != np.uint8:
            raise ValueError(f'expected a uint8 frame of shape {(self.H, self.W, 3)}, got {rgb.dtype} {rgb.shape}')
        self.qp = self.rc.qp
        Y, U, V = O.rgb_to_yuv420(rgb)
        k = self.n % self.gop
        idr = k == 0
        R, C = self.mbh, self.mbw
        if idr:
            mbs, rec = self._intra(Y, U, V)
            self.mvs, self.skip = None, None
            nz, mv = np.zeros((R, C, 4, 4), bool), np.zeros((R, C, 2), np.int64)
        else:
            mbs, rec = self._inter(Y, U, V)
            nz = np.zeros((R, C, 4, 4), bool)
            for k4, (bx, by) in enumerate(O.BLK):
                nz[:, :, by, bx] = [[np.any(mbs[r][c]['lac'][k4]) for c in range(C)] for r in range(R)]
            mv = self.mvs
        planes = tuple(p.swapaxes(1, 2).reshape(R * p.shape[2], C * p.shape[3]).astype(np.int64) for p in rec)
        deblock(planes, self.qp, *boundary_strength(idr, nz, mv))
        self.recon = tuple(p.astype(np.uint8) for p in planes)
        sample = b''.join(self._slice(r, mbs[r], idr, k % 16, (self.n // self.gop) % 2) for r in range(R))
        self.rc.update(len(sample), idr)
        self.qps.append(self.qp)
        self.n += 1
        return sample, idr


# ------------------------------------------------------------------------------------------------ test sequence
PAN = (1.25, -0.5)              # per-frame shift of the 'pan' sequence: frame t samples the pattern at x + 1.25t, y - 0.5t
PAN_SCALE = 3                   # ... with O._pattern's frequencies times 3 (at most 0.75 rad/sample per term), so that a quarter
                                # sample of motion moves the SAD well above the reconstruction's noise at QP 18


def pan(W, H, n=3):
    """n uint8 RGB frames [H, W, 3] of O._pattern's analytic pattern (frequencies scaled by PAN_SCALE) panned by a fraction of a
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


def frames(name, W, H, n=3):
    return pan(W, H, n) if name == 'pan' else O.sequence(name, W, H, n)
