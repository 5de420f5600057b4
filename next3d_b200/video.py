"""H.264 video on the device: `H264Encoder` encodes uint8 RGB frames with the sm_90a encoder of csrc/h264.cu into AVCC samples,
and `H264Writer` writes them to an MP4 file (next3d_b200.mp4).  The stream is Constrained Baseline (profile 66): 4:2:0 BT.601 limited range, CAVLC, one slice per macroblock
row, IDR frames of I_16x16 macroblocks, P frames of P_L0_16x16 / P_Skip.  Two streams (DESIGN.md section 3.5):
  * constant QP (the default): integer-pel motion, no deblocking;
  * with a `bitrate`: QP per picture from a rate controller on the device, quarter-sample motion and in-loop deblocking.
This module also writes the SPS and PPS, for the encoder and its numpy restatements alike; the slice headers are written by the
kernels."""
import fractions
import re

import numpy as np
import torch

from . import _lib, mp4

# Table A-1: level_idc, MaxMBPS, MaxFS (macroblocks).  Level 1b needs constraint_set3 and is skipped.
LEVELS = [(10, 1485, 99), (11, 3000, 396), (12, 6000, 396), (13, 11880, 396), (20, 11880, 396), (21, 19800, 792),
          (22, 20250, 1620), (30, 40500, 1620), (31, 108000, 3600), (32, 216000, 5120), (40, 245760, 8192), (41, 245760, 8192),
          (42, 522240, 8704), (50, 589824, 22080), (51, 983040, 36864), (52, 2073600, 36864), (60, 4177920, 139264),
          (61, 8355840, 139264), (62, 16711680, 139264)]
# Table A-1 MaxBR per level, in 1000 bits/s (cpbBrVclFactor of the Baseline profile)
MAX_BR = {10: 64, 11: 192, 12: 384, 13: 768, 20: 2000, 21: 4000, 22: 4000, 30: 10000, 31: 14000, 32: 20000, 40: 20000, 41: 50000,
          42: 50000, 50: 135000, 51: 240000, 52: 240000, 60: 240000, 61: 480000, 62: 800000}


def level_idc(width, height, fps, bitrate=None):
    """Smallest level whose MaxFS, MaxMBPS and frame-dimension limits (width, height <= sqrt(8 * MaxFS) macroblocks) fit, and
    with a bitrate (bits/s) its MaxBR."""
    mbw, mbh = (width + 15) // 16, (height + 15) // 16
    for lev, mbps, fs in LEVELS:
        if mbw * mbh <= fs and mbw * mbw <= 8 * fs and mbh * mbh <= 8 * fs and mbw * mbh * fps <= mbps and \
                (bitrate is None or bitrate <= 1000 * MAX_BR[lev]):
            return lev
    raise ValueError(f'{width}x{height} at {fps} frames/s' + ('' if bitrate is None else f' and {bitrate} bits/s')
                     + ' exceeds H.264 level 6.2')


def parse_bitrate(rate):
    """Bits/s from an int or an FFmpeg-style string ('10M', '800k', '1.5M', '2000000'); refuses a non-positive rate."""
    if isinstance(rate, str):
        m = re.fullmatch(r'\s*(\d+(?:\.\d*)?|\.\d+)\s*([kKMG]?)\s*', rate)
        if not m:
            raise ValueError(f'bitrate {rate!r}: expected bits/s such as 12000000, 800k or 10M')
        bits = round(float(m.group(1)) * {'': 1, 'k': 10 ** 3, 'K': 10 ** 3, 'M': 10 ** 6, 'G': 10 ** 9}[m.group(2)])
    elif isinstance(rate, (int, np.integer)) and not isinstance(rate, bool):
        bits = int(rate)
    else:
        raise ValueError(f'bitrate {rate!r}: expected an int (bits/s) or a string such as 10M')
    if bits <= 0:
        raise ValueError(f'bitrate must be positive, got {rate!r}')
    return bits


class _Bits:
    def __init__(self):
        self.s = []

    def u(self, v, n):
        self.s.append(format(int(v), f'0{n}b'))

    def ue(self, k):
        n = (k + 1).bit_length()
        self.s.append('0' * (n - 1))
        self.u(k + 1, n)

    def se(self, v):
        self.ue(2 * v - 1 if v > 0 else -2 * v)

    def nal(self, header):
        s = ''.join(self.s) + '1'
        s += '0' * (-len(s) % 8)
        rbsp = int(s, 2).to_bytes(len(s) // 8, 'big')
        out, zeros = bytearray([header]), 0
        for b in rbsp:                                   # emulation prevention
            if zeros >= 2 and b <= 3:
                out.append(3)
                zeros = 0
            out.append(b)
            zeros = zeros + 1 if b == 0 else 0
        return bytes(out)


def _fps_fraction(fps):
    f = fractions.Fraction(fps).limit_denominator(1001)
    if f <= 0:
        raise ValueError(f'fps must be positive, got {fps}')
    return f


def sps(width, height, fps, bitrate=None):
    """Sequence parameter set NAL unit (no start code); the level also covers `bitrate` (bits/s) when given."""
    mbw, mbh = (width + 15) // 16, (height + 15) // 16
    f = _fps_fraction(fps)
    b = _Bits()
    b.u(66, 8)                                       # profile_idc: Baseline
    b.u(0b11000000, 8)                               # constraint_set0/1: Constrained Baseline
    b.u(level_idc(width, height, float(f), bitrate), 8)
    b.ue(0)                                          # seq_parameter_set_id
    b.ue(0)                                          # log2_max_frame_num_minus4: frame_num is 4 bits
    b.ue(2)                                          # pic_order_cnt_type 2: output order = decoding order
    b.ue(1)                                          # max_num_ref_frames
    b.u(0, 1)                                        # gaps_in_frame_num_value_allowed_flag
    b.ue(mbw - 1)
    b.ue(mbh - 1)
    b.u(1, 1)                                        # frame_mbs_only_flag
    b.u(1, 1)                                        # direct_8x8_inference_flag
    crop = (mbw * 16 != width) or (mbh * 16 != height)
    b.u(crop, 1)
    if crop:                                         # in units of 2 samples (4:2:0, frames)
        b.ue(0)
        b.ue((mbw * 16 - width) // 2)
        b.ue(0)
        b.ue((mbh * 16 - height) // 2)
    b.u(1, 1)                                        # vui_parameters_present_flag
    b.u(0, 1)                                        # aspect_ratio_info_present_flag
    b.u(0, 1)                                        # overscan_info_present_flag
    b.u(1, 1)                                        # video_signal_type_present_flag
    b.u(5, 3)                                        # video_format: unspecified
    b.u(0, 1)                                        # video_full_range_flag: limited range
    b.u(1, 1)                                        # colour_description_present_flag
    b.u(6, 8)                                        # colour_primaries: SMPTE 170M
    b.u(6, 8)                                        # transfer_characteristics: SMPTE 170M
    b.u(6, 8)                                        # matrix_coefficients: BT.601
    b.u(0, 1)                                        # chroma_loc_info_present_flag
    b.u(1, 1)                                        # timing_info_present_flag
    b.u(f.denominator, 32)                           # num_units_in_tick
    b.u(2 * f.numerator, 32)                         # time_scale: two ticks per frame
    b.u(1, 1)                                        # fixed_frame_rate_flag
    b.u(0, 1)                                        # nal_hrd_parameters_present_flag
    b.u(0, 1)                                        # vcl_hrd_parameters_present_flag
    b.u(0, 1)                                        # pic_struct_present_flag
    b.u(1, 1)                                        # bitstream_restriction_flag
    b.u(1, 1)                                        # motion_vectors_over_pic_boundaries_flag
    b.ue(0)                                          # max_bytes_per_pic_denom: no limit
    b.ue(0)                                          # max_bits_per_mb_denom: no limit
    b.ue(16)                                         # log2_max_mv_length_horizontal
    b.ue(16)                                         # log2_max_mv_length_vertical
    b.ue(0)                                          # max_num_reorder_frames
    b.ue(1)                                          # max_dec_frame_buffering
    return b.nal(0x67)


def pps(qp):
    """Picture parameter set NAL unit: CAVLC, pic_init_qp = qp, deblocking control present (constant-QP slices disable the
    filter; the rate-controlled stream uses pps(26) and sets each slice's QP and filter)."""
    b = _Bits()
    b.ue(0)                                          # pic_parameter_set_id
    b.ue(0)                                          # seq_parameter_set_id
    b.u(0, 1)                                        # entropy_coding_mode_flag: CAVLC
    b.u(0, 1)                                        # bottom_field_pic_order_in_frame_present_flag
    b.ue(0)                                          # num_slice_groups_minus1
    b.ue(0)                                          # num_ref_idx_l0_default_active_minus1
    b.ue(0)                                          # num_ref_idx_l1_default_active_minus1
    b.u(0, 1)                                        # weighted_pred_flag
    b.u(0, 2)                                        # weighted_bipred_idc
    b.se(qp - 26)                                    # pic_init_qp_minus26
    b.se(0)                                          # pic_init_qs_minus26
    b.se(0)                                          # chroma_qp_index_offset
    b.u(1, 1)                                        # deblocking_filter_control_present_flag
    b.u(0, 1)                                        # constrained_intra_pred_flag
    b.u(0, 1)                                        # redundant_pic_cnt_present_flag
    return b.nal(0x68)


def check_args(width, height, fps, qp, gop, bitrate=None):
    if width <= 0 or height <= 0 or width % 2 or height % 2:
        raise ValueError(f'4:2:0 needs even, positive frame dimensions, got {width}x{height}')
    if not 0 <= qp <= 51:
        raise ValueError(f'qp must be in 0..51, got {qp}')
    if gop < 1:
        raise ValueError(f'gop must be at least 1, got {gop}')
    level_idc(width, height, float(_fps_fraction(fps)), bitrate)


class H264Encoder:
    """Encode uint8 RGB frames [H, W, 3] (numpy arrays or CUDA tensors, one frame or a batch [N, H, W, 3]) in order, on a stream
    of the encoder's own, and hand back the coded frames as (AVCC sample bytes, is_idr).  qp: constant quantiser 0..51 (lower =
    larger stream, closer to the input); gop: an IDR frame every `gop` frames.  CUDA frames are read in place; numpy frames are
    copied to the device.  The coded frames reach the host `batch` frames at a time in one pinned copy, one batch behind the
    encoder, so that the host does not wait for the frames it has just submitted: write() returns the samples finished so far
    (possibly none), flush() the rest.  `sps` and `pps` are the stream's parameter sets.

    bitrate (bits/s: an int, or a string such as '10M' or '800k'): the rate-controlled stream instead, with qp ignored.  Its
    controller runs on the device (no extra host synchronisation) and keeps each picture's QP within qp_range (min, max);
    equal bounds pin the QP.  `recon` is then the deblocked picture.

    first_frame (a multiple of gop): the index of the first frame in a longer video, which sets frame_num and idr_pic_id, so that
    encoders of consecutive ranges of a clip, split at multiples of gop, concatenate to the constant-QP stream of one encoder over
    the whole clip (nothing crosses an IDR frame).  A rate-controlled segment starts its own controller at the first QP."""

    def __init__(self, width, height, fps, qp=18, gop=60, device=None, batch=8, bitrate=None, qp_range=(0, 51), first_frame=0):
        self.bitrate = None if bitrate is None else parse_bitrate(bitrate)
        check_args(width, height, fps, qp, gop, self.bitrate)
        if first_frame < 0 or first_frame % gop:
            raise ValueError(f'first_frame must be a non-negative multiple of gop {gop}, got {first_frame}')
        qp_min, qp_max = (int(q) for q in qp_range)
        if not 0 <= qp_min <= qp_max <= 51:
            raise ValueError(f'qp_range must satisfy 0 <= min <= max <= 51, got {qp_range}')
        self.width, self.height, self.qp, self.gop, self.first_frame = int(width), int(height), int(qp), int(gop), int(first_frame)
        self.fps = _fps_fraction(fps)
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != 'cuda':
            raise ValueError('H264Encoder encodes on a CUDA device')
        sizes = [_lib.I64() for _ in range(4)]
        _lib.check(_lib.lib.n3d_h264_buffer_sizes(self.width, self.height, *[_lib.C.byref(s) for s in sizes]), 'n3d_h264_buffer_sizes')
        self.plane_bytes, scratch_bytes, slice_bytes, self.sample_cap = (s.value for s in sizes)
        mbw, mbh = (self.width + 15) // 16, (self.height + 15) // 16
        self._shape = (16 * mbh, 16 * mbw)
        self.stream = torch.cuda.Stream(self.device)
        self._copy = torch.cuda.Stream(self.device)                # sample read-back, off the encoder's stream
        self.batch = max(1, min(int(batch), (1 << 28) // self.sample_cap))          # two halves of at most 256 MB of samples
        with torch.cuda.device(self.device):
            new = lambda n: torch.empty(n, dtype=torch.uint8, device=self.device)
            self._cur, self._planes = new(self.plane_bytes), [new(self.plane_bytes), new(self.plane_bytes)]
            self._scratch, self._slices = new(scratch_bytes), new(slice_bytes)
            self._samples = new(2 * self.batch * self.sample_cap)
            self._lens = torch.zeros(2 * self.batch, dtype=torch.int64, device=self.device)
            self._rc = None
            if self.bitrate is not None:
                self._rc = torch.empty(_lib.H264_RC_STATE_BYTES // 8, dtype=torch.int64, device=self.device)
                self.stream.wait_stream(torch.cuda.current_stream(self.device))      # the allocation, before the encoder's stream
                _lib.check(_lib.lib.n3d_h264_rc_init(self._rc.data_ptr(), self.width, self.height, self.bitrate, self.fps.numerator,
                                                     self.fps.denominator, qp_min, qp_max, self.stream.cuda_stream), 'n3d_h264_rc_init')
        self._lens_host = torch.empty(2 * self.batch, dtype=torch.int64, pin_memory=True)
        self._host = torch.empty(0, dtype=torch.uint8)
        self._half = 0                                       # which half of the sample slots the next frames go to
        self._pending = []                                   # IDR flag of each frame encoded into the current half
        self._inflight = None                                # (half, IDR flags, event) of the submitted half not yet read back
        self._done = []                                      # (sample, is_idr) read back and not yet handed out
        self.frames = 0
        self.sps = sps(self.width, self.height, fps, self.bitrate)
        self.pps = pps(self.qp if self._rc is None else 26)

    def write(self, frames):
        """Encode the frames; -> [(sample bytes, is_idr)] of the frames finished so far, in order."""
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(np.ascontiguousarray(frames))
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
            raise TypeError('frames must be uint8 numpy arrays or tensors')
        if frames.dim() == 3:
            frames = frames[None]
        if tuple(frames.shape[1:]) != (self.height, self.width, 3):
            raise ValueError(f'expected frames of shape [N, {self.height}, {self.width}, 3], got {list(frames.shape)}')
        producer = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self.stream):
            if frames.device != self.device:
                frames = frames.to(self.device)                   # numpy / host frames: copied on the encoder's stream
            else:
                self.stream.wait_stream(producer)                 # CUDA frames: read in place once their producer is done
                frames.record_stream(self.stream)
            frames = frames.contiguous()
            for i in range(frames.shape[0]):
                self._encode(frames[i])
        return self._take()

    def flush(self):
        """Wait for every frame written so far; -> [(sample bytes, is_idr)] of those not yet returned, in order."""
        self._submit()
        self._read_back()
        return self._take()

    def _take(self):
        out, self._done = self._done, []
        return out

    def _encode(self, frame):
        n = self.first_frame + self.frames                       # index of the frame in the whole video
        k = n % self.gop
        slot = self._half * self.batch + len(self._pending)
        ref, rec = self._planes[self.frames % 2], self._planes[(self.frames + 1) % 2]
        fn, name = ((_lib.lib.n3d_h264_encode, 'n3d_h264_encode') if self._rc is None else
                    (_lib.lib.n3d_h264_encode_rc, 'n3d_h264_encode_rc'))
        _lib.check(fn(
            frame.data_ptr(), self.width, self.height, self.qp if self._rc is None else self._rc.data_ptr(), int(k == 0), k % 16,
            (n // self.gop) % 2, self._cur.data_ptr(), None if k == 0 else ref.data_ptr(), rec.data_ptr(),
            self._scratch.data_ptr(), self._slices.data_ptr(), self._samples[slot * self.sample_cap:].data_ptr(),
            self._lens[slot:].data_ptr(), self.stream.cuda_stream), name)
        self._pending.append(k == 0)
        self.frames += 1
        if len(self._pending) == self.batch:
            self._submit()

    def _submit(self):
        """Close the current half: its lengths go to the host behind its frames on the encoder's stream; the half submitted
        before it is read back (its frames were queued a batch earlier), so that its slots are free for the next frames."""
        n = len(self._pending)
        if n == 0:
            return
        o = self._half * self.batch
        with torch.cuda.stream(self.stream):
            self._lens_host[o:o + n].copy_(self._lens[o:o + n], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self._read_back()
        self._inflight = (self._half, self._pending, ev)
        self._pending = []
        self._half ^= 1

    def _read_back(self):
        if self._inflight is None:
            return
        h, idrs, ev = self._inflight
        self._inflight = None
        o, n = h * self.batch, len(idrs)
        ev.synchronize()
        lens = self._lens_host[o:o + n].tolist()
        if min(lens) < 0:
            raise RuntimeError('n3d_h264_encode: a slice exceeded its bitstream capacity')
        if self._host.numel() < sum(lens):
            self._host = torch.empty(max(sum(lens), 2 * self._host.numel()), dtype=torch.uint8, pin_memory=True)
        self._copy.wait_event(ev)
        with torch.cuda.stream(self._copy):
            p = 0
            for i, ln in enumerate(lens):
                s = (o + i) * self.sample_cap
                self._host[p:p + ln].copy_(self._samples[s:s + ln], non_blocking=True)
                p += ln
        self._copy.synchronize()
        data = self._host[:p].numpy().tobytes()
        p = 0
        for ln, idr in zip(lens, idrs):
            self._done.append((data[p:p + ln], idr))
            p += ln

    @property
    def recon(self):
        """Reconstruction of the last frame, as the decoder outputs it before cropping (deblocked in the rate-controlled
        stream): padded (Y [H16, W16], Cb, Cr [H16/2, W16/2]) uint8 CUDA tensors (copies)."""
        if self.frames == 0:
            return None
        self.stream.synchronize()
        p = self._planes[self.frames % 2]
        H16, W16 = self._shape
        n = H16 * W16
        return (p[:n].view(H16, W16).clone(), p[n:n + n // 4].view(H16 // 2, W16 // 2).clone(),
                p[n + n // 4:n + n // 2].view(H16 // 2, W16 // 2).clone())


class H264Writer(H264Encoder):
    """H264Encoder into an MP4 file at `path` (next3d_b200.mp4.Mp4Writer): every coded frame goes to the file as soon as it is
    back on the host.  Arguments as H264Encoder's.  Use as a context manager, or call close()."""

    def __init__(self, path, width, height, fps, qp=18, gop=60, device=None, batch=8, bitrate=None, qp_range=(0, 51), first_frame=0):
        super().__init__(width, height, fps, qp=qp, gop=gop, device=device, batch=batch, bitrate=bitrate, qp_range=qp_range,
                         first_frame=first_frame)
        self._mp4 = mp4.Mp4Writer(path, self.width, self.height, self.fps, self.sps, self.pps)

    def write(self, frames):
        for sample, idr in super().write(frames):
            self._mp4.add(sample, idr)

    def close(self):
        if self._mp4 is None:
            return
        try:
            for sample, idr in self.flush():
                self._mp4.add(sample, idr)
        finally:
            self._mp4.close()
            self._mp4 = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
