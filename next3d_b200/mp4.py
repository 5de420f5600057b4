"""Write an H.264 elementary stream as an MP4 file (ISO/IEC 14496-12 and -15): `ftyp`, `mdat` with the samples, then `moov` with
one video track.  Samples are AVCC access units (4-byte big-endian NAL lengths), as next3d_b200.video produces them."""
import struct

TIMESCALE = 90000                        # media timescale of the track; the movie timescale is 1000


def box(kind, *payload):
    data = b''.join(payload)
    return struct.pack('>I4s', 8 + len(data), kind) + data


def full_box(kind, version, flags, *payload):
    return box(kind, struct.pack('>I', (version << 24) | flags), *payload)


def _matrix():
    return struct.pack('>9I', 0x10000, 0, 0, 0, 0x10000, 0, 0, 0, 0x40000000)


def avcc(sps, pps):
    """AVCDecoderConfigurationRecord with one SPS and one PPS (NAL units without start codes or lengths)."""
    return box(b'avcC', bytes([1, sps[1], sps[2], sps[3], 0xff, 0xe1]), struct.pack('>H', len(sps)), sps,
               bytes([1]), struct.pack('>H', len(pps)), pps)


class Mp4Writer:
    """Streams AVCC samples into `mdat` as they come and writes `moov` on close().  fps: frames per second (a number or a
    Fraction); every sample lasts TIMESCALE / fps ticks, which must be a whole number."""

    def __init__(self, path, width, height, fps, sps, pps):
        delta = TIMESCALE / fps
        if delta != int(delta) or delta <= 0:
            raise ValueError(f'{fps} frames/s is not a whole number of {TIMESCALE} Hz ticks')
        self.delta, self.width, self.height, self.sps, self.pps = int(delta), width, height, sps, pps
        self.sizes, self.sync = [], []
        self.f = open(path, 'wb')
        self.f.write(box(b'ftyp', b'isom', struct.pack('>I', 0x200), b'isom', b'iso2', b'avc1', b'mp41'))
        self.mdat = self.f.tell()
        self.f.write(struct.pack('>I4sQ', 1, b'mdat', 0))          # 64-bit size, patched in close()
        self.offset = self.f.tell()

    def add(self, sample, sync):
        if sync:
            self.sync.append(len(self.sizes))
        self.sizes.append(len(sample))
        self.f.write(sample)

    def close(self):
        if self.f is None:
            return
        f, self.f = self.f, None
        try:
            end = f.tell()
            f.seek(self.mdat + 8)
            f.write(struct.pack('>Q', end - self.mdat))
            f.seek(end)
            f.write(self._moov())
        finally:
            f.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _moov(self):
        n, delta, width, height = len(self.sizes), self.delta, self.width, self.height
        duration_media = n * delta
        duration_movie = duration_media * 1000 // TIMESCALE
        avc1 = box(b'avc1', bytes(6), struct.pack('>H', 1), bytes(16), struct.pack('>HH', width, height),
                   struct.pack('>II', 0x480000, 0x480000), bytes(4), struct.pack('>H', 1), bytes(32),
                   struct.pack('>Hh', 0x18, -1), avcc(self.sps, self.pps))
        stsd = full_box(b'stsd', 0, 0, struct.pack('>I', 1), avc1)
        stts = full_box(b'stts', 0, 0, struct.pack('>III', 1, n, delta))
        stss = full_box(b'stss', 0, 0, struct.pack('>I', len(self.sync)), b''.join(struct.pack('>I', i + 1) for i in self.sync))
        stsz = full_box(b'stsz', 0, 0, struct.pack('>II', 0, n), b''.join(struct.pack('>I', s) for s in self.sizes))
        stsc = full_box(b'stsc', 0, 0, struct.pack('>IIII', 1, 1, 1, 1))          # one sample per chunk
        offs, o = [], self.offset
        for s in self.sizes:
            offs.append(o)
            o += s
        if o > 0xffffffff:
            stco = full_box(b'co64', 0, 0, struct.pack('>I', n), b''.join(struct.pack('>Q', x) for x in offs))
        else:
            stco = full_box(b'stco', 0, 0, struct.pack('>I', n), b''.join(struct.pack('>I', x) for x in offs))
        stbl = box(b'stbl', stsd, stts, stss, stsz, stsc, stco)
        dinf = box(b'dinf', full_box(b'dref', 0, 0, struct.pack('>I', 1), full_box(b'url ', 0, 1)))
        minf = box(b'minf', full_box(b'vmhd', 0, 1, bytes(8)), dinf, stbl)
        hdlr = full_box(b'hdlr', 0, 0, bytes(4), b'vide', bytes(12), b'VideoHandler\x00')
        mdhd = full_box(b'mdhd', 0, 0, struct.pack('>IIIIHH', 0, 0, TIMESCALE, duration_media, 0x55c4, 0))   # language 'und'
        mdia = box(b'mdia', mdhd, hdlr, minf)
        tkhd = full_box(b'tkhd', 0, 3, struct.pack('>IIIII', 0, 0, 1, 0, duration_movie), bytes(8),
                        struct.pack('>hhhH', 0, 0, 0, 0), _matrix(), struct.pack('>II', width << 16, height << 16))
        mvhd = full_box(b'mvhd', 0, 0, struct.pack('>IIII', 0, 0, 1000, duration_movie), struct.pack('>IH', 0x10000, 0x100),
                        bytes(10), _matrix(), bytes(24), struct.pack('>I', 2))
        return box(b'moov', mvhd, box(b'trak', tkhd, mdia))


def write_mp4(path, width, height, fps, sps, pps, samples, sync):
    """All samples at once: samples is a list of AVCC access units, sync the 0-based indices of the IDR ones."""
    sync = set(sync)
    with Mp4Writer(path, width, height, fps, sps, pps) as w:
        for i, s in enumerate(samples):
            w.add(s, i in sync)


def parse_boxes(data, start=0, end=None):
    """[(type, payload start, payload end)] of the boxes in data[start:end] (no recursion)."""
    end = len(data) if end is None else end
    out = []
    while start < end:
        size, kind = struct.unpack('>I4s', data[start:start + 8])
        head = 8
        if size == 1:
            size = struct.unpack('>Q', data[start + 8:start + 16])[0]
            head = 16
        elif size == 0:
            size = end - start
        out.append((kind, start + head, start + size))
        start += size
    return out
