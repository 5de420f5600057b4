"""Per-frame inputs of the inference scripts (SURVEY.md section 8, row f3): the FLAME mesh (.obj) and the 68 2-D landmarks
(*_kpt2d.txt) that `gen_samples_next3d.py:165-178`, `gen_videos_next3d.py:118-131` and `reenact_avatar_next3d.py:128-141`
parse in Python for every frame, plus a prefetcher that keeps parsed frames in pinned host memory ahead of the generator.

The parsers are native (`n3d_parse_obj_vertices`, `n3d_parse_float_table` in libnext3d_b200.so): one pass over the file, values
bit-identical to the reference's `float(token)` -> float64 -> `.float()`.
Also here: the `dataset.json` camera labels of the reenactment script (reenact_avatar_next3d.py:110-111,159) and a binary frame
pack (all meshes + cameras of a driving sequence in one memory-mappable file) so that a clip is parsed once, not per run.
"""
import concurrent.futures
import copy
import ctypes as C
import json
import os

import numpy as np
import torch

from . import _lib


def _read(path_or_bytes):
    return bytes(path_or_bytes) if isinstance(path_or_bytes, (bytes, bytearray)) else open(path_or_bytes, 'rb').read()


def _err():
    return ValueError(_lib.lib.n3d_last_error().decode())


def load_obj_vertices(path_or_bytes):
    """-> float32 [V, 3]: the `v ` lines of a Wavefront .obj (gen_samples_next3d.py:165-174)."""
    data = _read(path_or_bytes)
    cap = len(data) // 6 + 1                        # a vertex line is at least "v 0 0 0": one pass, no sizing pass
    out = np.empty((cap, 3), np.float32)
    n = C.c_int64(0)
    if _lib.lib.n3d_parse_obj_vertices(data, len(data), out.ctypes.data, cap, C.byref(n)) != 0:
        raise _err()
    return out[: n.value].copy() if n.value * 4 < cap else out[: n.value]


def load_float_table(path_or_bytes):
    """-> float32 [rows, cols] (1-D for a single row, like np.loadtxt): whitespace-separated numbers, '#' comments."""
    data = _read(path_or_bytes)
    cap = len(data) // 2 + 1                        # a number and its separator take at least two bytes
    out = np.empty(cap, np.float32)
    n, cols = C.c_int64(0), C.c_int64(0)
    if _lib.lib.n3d_parse_float_table(data, len(data), out.ctypes.data, cap, C.byref(n), C.byref(cols)) != 0:
        raise _err()
    out = out[: n.value].copy()
    if cols.value == 0:
        return out
    rows = n.value // cols.value
    return out.reshape(rows, cols.value) if rows > 1 else out


def load_frame(obj_path, lms_path=None, pin=False):
    """-> `v` as `TriPlaneGenerator.synthesis` takes it: float32 [1, V (+ 68), 3] = vertices, then the landmarks
    (gen_samples_next3d.py:165-178: `torch.cat((v, lms), 1)`).  pin=True returns page-locked memory (async H2D)."""
    parts = [load_obj_vertices(obj_path)]
    if lms_path is not None:
        lms = load_float_table(lms_path)
        parts.append(np.asarray(lms, np.float32).reshape(-1, parts[0].shape[1]))
    t = torch.from_numpy(np.concatenate(parts, 0))[None]
    return t.pin_memory() if pin else t


def load_photo(png_path, size=512, pin=False):
    """-> uint8 [size, size, 3] tensor: `np.array(Image.open(png).crop((0, 0, size, size)))`, the driving photo of
    reenact_avatar_next3d.py:132-133 (pixels outside the image read as 0, as PIL's crop gives them).  pin=True: page-locked."""
    from PIL import Image
    with Image.open(png_path) as im:
        a = np.array(im.crop((0, 0, size, size)))
    if a.ndim != 3 or a.shape[2] != 3:
        raise ValueError(f'{png_path}: the driving photo must be an RGB image, got array shape {a.shape}')
    t = torch.from_numpy(a)
    return t.pin_memory() if pin else t


class FramePrefetcher:
    """Iterate over (obj_path, lms_path) pairs, parsing `depth` frames ahead on worker threads (the parsers release the GIL
    inside the native call) and yielding pinned `[1, V+68, 3]` tensors in order.  With `photos` (one PNG path per frame) every
    item is (mesh, photo), the photo decoded by load_photo on the same worker threads."""

    def __init__(self, frames, depth=4, workers=2, pin=None, photos=None):
        self.frames = list(frames)
        self.photos = None if photos is None else list(photos)
        if self.photos is not None and len(self.photos) != len(self.frames):
            raise ValueError(f'FramePrefetcher: {len(self.photos)} photos for {len(self.frames)} frames')
        self.depth = max(1, depth)
        self.pin = torch.cuda.is_available() if pin is None else pin
        self.pool = concurrent.futures.ThreadPoolExecutor(max_workers=workers)

    def __len__(self):
        return len(self.frames)

    def _load(self, i):
        f = self.frames[i]
        mesh = load_frame(f[0], f[1], self.pin)
        return mesh if self.photos is None else (mesh, load_photo(self.photos[i], pin=self.pin))

    def __iter__(self):
        pending = []
        it = iter(range(len(self.frames)))
        try:
            for _ in range(self.depth):
                i = next(it, None)
                if i is None:
                    break
                pending.append(self.pool.submit(self._load, i))
            while pending:
                out = pending.pop(0).result()
                i = next(it, None)
                if i is not None:
                    pending.append(self.pool.submit(self._load, i))
                yield out
        finally:
            for p in pending:
                p.cancel()


# ------------------------------------------------------------------------------------------------ dataset.json labels
def load_labels(dataset_json):
    """`json.load(f)['labels']` of a driving sequence (reenact_avatar_next3d.py:110-111): list of [file name, 25 camera floats]."""
    with open(dataset_json, 'rb') as f:
        return json.load(f)['labels']


def smoothed_cameras(labels, ks):
    """Camera of frame k as the script computes it (reenact_avatar_next3d.py:159-160): the mean of the labels of frames k-1, k,
    k+1 in float64, then `.float()`.  -> float32 [len(ks), 25]."""
    out = [(np.array(labels[k - 1][1]) + np.array(labels[k][1]) + np.array(labels[k + 1][1])) / 3 for k in ks]
    return torch.tensor(np.stack(out)).float() if out else torch.zeros(0, 25)


# ------------------------------------------------------------------------------------------------ binary frame pack
_PACK_MAGIC = b'N3DPACK1'


def write_frame_pack(path, verts, cams, ids=None):
    """One file for a whole driving sequence: header (magic, F, V, json of the frame ids) + float32 verts [F, V, 3] + float32
    cams [F, 25], both 64-byte aligned so that they can be memory-mapped and copied to the device without parsing."""
    verts = np.ascontiguousarray(np.asarray(verts, np.float32))
    cams = np.ascontiguousarray(np.asarray(cams, np.float32))
    F_, V = verts.shape[0], verts.shape[1]
    assert verts.shape == (F_, V, 3) and cams.shape == (F_, 25)
    meta = json.dumps({'ids': list(ids) if ids is not None else None}).encode()
    head = _PACK_MAGIC + np.array([F_, V, len(meta)], np.int64).tobytes() + meta
    head += b'\0' * (-len(head) % 64)
    with open(path, 'wb') as f:
        f.write(head)
        f.write(verts.tobytes())
        f.write(b'\0' * (-verts.nbytes % 64))
        f.write(cams.tobytes())


class FramePack:
    """Memory-mapped reader of write_frame_pack files: `.verts` [F, V, 3], `.cams` [F, 25] (numpy memmaps), `.ids`;
    iterating yields pinned `[1, V, 3]` tensors in order (drop-in for FramePrefetcher in drivers.render_frames); `pack[a:b]` is
    the same reader over frames a .. b-1 (one rank's share of a clip)."""

    def __init__(self, path, pin=None):
        with open(path, 'rb') as f:
            if f.read(8) != _PACK_MAGIC:
                raise ValueError(f'{path}: not a next3d_b200 frame pack')
            F_, V, nmeta = (int(x) for x in np.frombuffer(f.read(24), np.int64))
            self.ids = json.loads(f.read(nmeta).decode())['ids']
        off = 8 + 24 + nmeta
        off += -off % 64
        self.verts = np.memmap(path, np.float32, 'r', off, (F_, V, 3))
        off += self.verts.nbytes + (-self.verts.nbytes % 64)
        self.cams = np.memmap(path, np.float32, 'r', off, (F_, 25))
        self.pin = torch.cuda.is_available() if pin is None else pin

    def __len__(self):
        return self.verts.shape[0]

    def __getitem__(self, frames):
        """pack[a:b]: the frames a .. b-1 as a FramePack over the same mapping (nothing is read until iterated)."""
        if not isinstance(frames, slice) or frames.step not in (None, 1):
            raise TypeError('FramePack supports contiguous slices only (pack[a:b])')
        view = copy.copy(self)
        view.verts, view.cams = self.verts[frames], self.cams[frames]
        view.ids = self.ids[frames] if self.ids is not None else None
        return view

    def __iter__(self):
        for i in range(len(self)):
            t = torch.from_numpy(np.array(self.verts[i]))[None]
            yield t.pin_memory() if self.pin else t
