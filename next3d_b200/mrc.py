"""Write a density grid as an MRC2014 map (the `.mrc` shapes of gen_samples_next3d.py:244-246, viewable in ChimeraX), and read
such maps back (the input of the shape_utils command)."""
import os

import numpy as np

HEADER_BYTES = 1024


def read_mrc(path):
    """The float32 data [nz, ny, nx] of an MRC map, memory-mapped (copy-on-write): what write_mrc writes and what mrcfile's
    new_mmap(..., mrc_mode=2) writes.  The extended header (NSYMBT bytes) is skipped.  ValueError, naming the field, for
    anything else: a mode other than 2, a machine stamp other than little-endian, an axis order other than 1, 2, 3, or a file
    shorter than its header says."""
    size = os.path.getsize(path)
    if size < HEADER_BYTES:
        raise ValueError(f'{path}: {size} bytes, shorter than the {HEADER_BYTES}-byte MRC header')
    with open(path, 'rb') as f:
        raw = f.read(HEADER_BYTES)
    stamp = raw[212:214]
    if stamp not in (b'\x44\x44', b'\x44\x41'):
        raise ValueError(f'{path}: machine stamp {raw[212:216].hex()} is not little-endian (44 44 00 00 or 44 41 00 00)')
    h = np.frombuffer(raw, '<i4')
    nx, ny, nz = (int(v) for v in h[0:3])
    if h[3] != 2:
        raise ValueError(f'{path}: mode {h[3]}: only mode 2 (float32) is read')
    if tuple(h[16:19]) != (1, 2, 3):
        raise ValueError(f'{path}: map order (mapc, mapr, maps) = {tuple(int(v) for v in h[16:19])}: only 1, 2, 3 is read')
    if min(nx, ny, nz) < 1:
        raise ValueError(f'{path}: dimensions (nx, ny, nz) = ({nx}, {ny}, {nz}) must be positive')
    if h[23] < 0:
        raise ValueError(f'{path}: nsymbt {h[23]} is negative')
    offset = HEADER_BYTES + int(h[23])
    if size < offset + 4 * nx * ny * nz:
        raise ValueError(f'{path}: truncated: {size} bytes, the header (nx, ny, nz, nsymbt) = ({nx}, {ny}, {nz}, {h[23]}) needs '
                         f'{offset + 4 * nx * ny * nz}')
    return np.memmap(path, dtype='<f4', mode='c', offset=offset, shape=(nz, ny, nx))


def write_mrc(path, data):
    """Write float32 data [nz, ny, nx] as an MRC2014 file: mode 2 (float32), a cell as large as the grid (voxel size 1), axis order
    x, y, z (mapc/mapr/maps 1/2/3), dmin / dmax / dmean / rms of the data, and the little-endian machine stamp."""
    data = np.ascontiguousarray(data, dtype='<f4')
    if data.ndim != 3:
        raise ValueError(f'an MRC map is a 3-D grid, got shape {data.shape}')
    nz, ny, nx = data.shape
    d64 = data.astype(np.float64)
    header = np.zeros(256, dtype='<i4')
    words = header.view('<f4')
    header[0:3] = nx, ny, nz
    header[3] = 2                                        # mode 2: 32-bit float
    header[7:10] = nx, ny, nz                            # mx, my, mz: sampling intervals along the cell
    words[10:13] = nx, ny, nz                            # cell dimensions (angstroms): one unit per voxel
    words[13:16] = 90.0                                  # cell angles
    header[16:19] = 1, 2, 3                              # columns, rows, sections = x, y, z
    words[19:22] = d64.min(), d64.max(), d64.mean()
    header[22] = 1                                       # space group 1: a single volume
    header[27] = 20140                                   # format version MRC2014
    header[52] = int.from_bytes(b'MAP ', 'little')
    header[53] = int.from_bytes(bytes([0x44, 0x44, 0, 0]), 'little')   # machine stamp: little-endian
    words[54] = d64.std()                                # rms deviation from the mean
    with open(path, 'wb') as f:
        f.write(header.tobytes())
        f.write(data.tobytes())
