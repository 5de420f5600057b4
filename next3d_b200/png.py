"""PNG images on the device: `PngEncoder` encodes batches of uint8 RGB images with the sm_90a encoder of csrc/png.cu into PNG
files (8-bit RGB, no interlace), and `encode_png` is its one-call form.  A file's bytes are a function of its pixels alone
(DESIGN.md section 3.6; tests/png_oracle.py restates the encoder in numpy)."""
import numpy as np
import torch

from . import _lib


def check_args(width, height, batch=1):
    if width <= 0 or height <= 0:
        raise ValueError(f'PNG images need positive dimensions, got {width}x{height}')
    if batch < 1:
        raise ValueError(f'batch must be at least 1, got {batch}')
    scratch, cap = _lib.I64(), _lib.I64()
    _lib.check(_lib.lib.n3d_png_buffer_sizes(int(batch), int(height), int(width), _lib.C.byref(scratch), _lib.C.byref(cap)),
               'n3d_png_buffer_sizes')
    return scratch.value, cap.value


class PngEncoder:
    """Encode uint8 RGB images [H, W, 3] (numpy arrays or CUDA tensors, one image or a batch [N, H, W, 3]) in order, on a stream
    of the encoder's own, and hand back the PNG files as bytes.  CUDA images are read in place; numpy images are copied to the
    device.  Up to `batch` images are encoded per launch; the files reach the host a batch at a time in one pinned copy, one
    batch behind the encoder, so that the host does not wait for the images it has just submitted: write() returns the files
    finished so far (possibly none), flush() the rest."""

    def __init__(self, width, height, device=None, batch=8):
        self.width, self.height = int(width), int(height)
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != 'cuda':
            raise ValueError('PngEncoder encodes on a CUDA device')
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        _, self.file_cap = check_args(self.width, self.height)
        self.batch = max(1, min(int(batch), (1 << 28) // self.file_cap))          # two halves of at most 256 MB of files
        scratch_bytes, _ = check_args(self.width, self.height, self.batch)
        self.stream = torch.cuda.Stream(self.device)
        self._copy = torch.cuda.Stream(self.device)                   # file read-back, off the encoder's stream
        with torch.cuda.device(self.device):
            self._scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=self.device)
            self._files = torch.empty(2 * self.batch * self.file_cap, dtype=torch.uint8, device=self.device)
            self._lens = torch.zeros(2 * self.batch, dtype=torch.int64, device=self.device)
        self._lens_host = torch.empty(2 * self.batch, dtype=torch.int64, pin_memory=True)
        self._host = torch.empty(0, dtype=torch.uint8)
        self._half = 0                   # which half of the file slots the next images go to
        self._pending = 0                # images encoded into the current half
        self._inflight = None            # (half, count, event) of the submitted half not yet read back
        self._done = []                  # files read back and not yet handed out
        self.images = 0

    def write(self, frames):
        """Encode the images; -> [bytes] of the PNG files finished so far, in order."""
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(np.ascontiguousarray(frames))
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
            raise TypeError('images must be uint8 numpy arrays or tensors')
        if frames.dim() == 3:
            frames = frames[None]
        if frames.dim() != 4 or tuple(frames.shape[1:]) != (self.height, self.width, 3):
            raise ValueError(f'expected images of shape [N, {self.height}, {self.width}, 3], got {list(frames.shape)}')
        if frames.device.type == 'cuda' and frames.device != self.device:
            raise ValueError(f'images are on {frames.device}, the encoder on {self.device}')
        producer = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self.stream):
            if frames.device != self.device:
                frames = frames.to(self.device)                   # numpy / host images: copied on the encoder's stream
            else:
                self.stream.wait_stream(producer)                 # CUDA images: read in place once their producer is done
                frames.record_stream(self.stream)
            frames = frames.contiguous()
            i = 0
            while i < frames.shape[0]:
                k = min(frames.shape[0] - i, self.batch - self._pending)
                slot = self._half * self.batch + self._pending
                _lib.check(_lib.lib.n3d_png_encode(
                    frames[i].data_ptr(), k, self.height, self.width, self._scratch.data_ptr(),
                    self._files[slot * self.file_cap:].data_ptr(), self._lens[slot:].data_ptr(), self.stream.cuda_stream),
                    'n3d_png_encode')
                i += k
                self._pending += k
                self.images += k
                if self._pending == self.batch:
                    self._submit()
        return self._take()

    def flush(self):
        """Wait for every image written so far; -> [bytes] of the files not yet returned, in order."""
        self._submit()
        self._read_back()
        return self._take()

    def _take(self):
        out, self._done = self._done, []
        return out

    def _submit(self):
        """Close the current half: its lengths go to the host behind its images on the encoder's stream; the half submitted
        before it is read back, so that its slots are free for the next images."""
        n = self._pending
        if n == 0:
            return
        o = self._half * self.batch
        with torch.cuda.stream(self.stream):
            self._lens_host[o:o + n].copy_(self._lens[o:o + n], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self._read_back()
        self._inflight = (self._half, n, ev)
        self._pending = 0
        self._half ^= 1

    def _read_back(self):
        if self._inflight is None:
            return
        h, n, ev = self._inflight
        self._inflight = None
        o = h * self.batch
        ev.synchronize()
        lens = self._lens_host[o:o + n].tolist()
        if self._host.numel() < sum(lens):
            self._host = torch.empty(max(sum(lens), 2 * self._host.numel()), dtype=torch.uint8, pin_memory=True)
        self._copy.wait_event(ev)
        with torch.cuda.stream(self._copy):
            p = 0
            for i, ln in enumerate(lens):
                s = (o + i) * self.file_cap
                self._host[p:p + ln].copy_(self._files[s:s + ln], non_blocking=True)
                p += ln
        self._copy.synchronize()
        data = self._host[:p].numpy().tobytes()
        p = 0
        for ln in lens:
            self._done.append(data[p:p + ln])
            p += ln


def encode_png(frames, device=None, batch=8):
    """uint8 RGB images [N, H, W, 3] (or one [H, W, 3]; numpy or CUDA) -> list of PNG file bytes, one per image."""
    if not isinstance(frames, (np.ndarray, torch.Tensor)):
        raise TypeError('images must be uint8 numpy arrays or tensors')
    if frames.ndim == 3:
        frames = frames[None]
    if frames.ndim != 4 or frames.shape[3] != 3:
        raise ValueError(f'expected images of shape [N, H, W, 3], got {list(frames.shape)}')
    if device is None and isinstance(frames, torch.Tensor) and frames.is_cuda:
        device = frames.device
    enc = PngEncoder(frames.shape[2], frames.shape[1], device=device, batch=batch)
    return enc.write(frames) + enc.flush()
