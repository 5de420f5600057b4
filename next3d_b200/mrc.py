"""Write a density grid as an MRC2014 map (the `.mrc` shapes of gen_samples_next3d.py:244-246, viewable in ChimeraX)."""
import numpy as np


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
