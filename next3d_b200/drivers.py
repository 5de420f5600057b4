"""Batched frame drivers (SURVEY.md section 8, row f1): the per-frame Python loops of `gen_videos_next3d.py:128-171`,
`reenact_avatar_next3d.py:125-167` and `gen_samples_next3d.py:182-238` restated as (1) a schedule computed up front -- orbit cameras,
interpolated latents, driving frames -- and (2) a loop over BATCHES of frames through `TriPlaneGenerator.synthesis` (CUDA-graph
replay) or `render_views`, with the uint8 conversion on the device, so that nothing but the generator sits on the critical path.

Each workload (interpolated frames, one-head orbits, reenactment, the two grids, sample sheets) is written once, as a private
function that does its setup and returns `step(k, idx)`: render step k of a plan (ShardPlan), the frames idx, and return their
uint8 frames.  Its two public drivers differ only in the plan and in how the finished batches leave the device: the single-process
generator (local_plan: exactly `batch` frames per step) streams them to the caller through _to_host, an asynchronous read-back
under the next step; the sharded twin (shard_plan: one process per GPU, contiguous frame ranges) gathers them to rank 0 through
_gather_frames.  The sampler keywords of every call follow one rule (_sampler_kw).  The CLI's videos under torchrun use a third
plan, CallPlan: each rank makes exactly the single-process calls that hold its own whole GOPs (the *_video_shard drivers), and
write_video_sharded encodes them on its GPU and gathers only the coded samples to rank 0.

Three outputs render heads in several views -- sample sheets, multi-view datasets (render_dataset) and coloured meshes
(coloured_meshes) -- and share one step, _head_views_step: view 0 of the call's heads through a caching synthesis call, the other
views through one render_views call, with sampler seed ids 2 c and 2 c + 1 for call c.  Their cameras come from one builder
(_view_cameras).  The CLI splits their heads over ranks with one plan, head_plan: a CallPlan of whole calls, so each rank makes
single-process calls and keeps every head of them (the sheets' sharded twin keeps shard_plan).

Everything here is host logic around the hot path; the per-frame values (camera matrices, interpolated ws, uint8 pixels) are the
reference's, checked in tests/test_drivers_cpu.py against the reference's own code, and the calls every driver makes in
tests/test_driver_calls_cpu.py.
"""
from typing import NamedTuple

import numpy as np
import torch

from . import camera

FOCAL_FFHQ = 4.2647            # gen_videos_next3d.py:97,139


def orbit_camera_params(num_frames, lookat, radius, yaw_range=0.35, pitch_range=0.25, focal=FOCAL_FFHQ):
    """-> c [num_frames, 25] float32: the camera sweep of gen_videos_next3d.py:128-140 (note the script's 3.14 literals)."""
    intr = torch.tensor([[focal, 0, 0.5], [0, focal, 0.5], [0, 0, 1]], dtype=torch.float32)
    half = num_frames // 2
    out = []
    for f in range(num_frames):
        pose = camera.look_at_pose(3.14 / 2 + yaw_range * np.sin(2 * 3.14 * f / half),
                                   3.14 / 2 - 0.05 + pitch_range * np.cos(2 * 3.14 * f / half), lookat, radius)
        out.append(torch.cat([pose.reshape(16), intr.reshape(9)]))
    return torch.stack(out)


def interpolate_ws(ws_keyframes, w_frames, wraps=2, kind='cubic'):
    """ws_keyframes [K, L, D] (one grid cell of gen_videos_next3d.py:106-117) -> [K * w_frames, L, D]: the latents of every
    frame, `interp(frame_idx / w_frames)` for frame_idx = 0 .. K*w_frames-1 (:143-144), evaluated in one call."""
    import scipy.interpolate
    K = ws_keyframes.shape[0]
    x = np.arange(-K * wraps, K * (wraps + 1))
    y = np.tile(ws_keyframes.detach().cpu().numpy(), [wraps * 2 + 1, 1, 1])
    interp = scipy.interpolate.interp1d(x, y, kind=kind, axis=0)
    return torch.from_numpy(interp(np.arange(K * w_frames) / w_frames))


def to_uint8_hwc(img):
    """[N,3,H,W] float in [-1,1] -> [N,H,W,3] uint8, the arithmetic of layout_grid (gen_videos_next3d.py:40-46) for a 1x1 grid."""
    return (img * 127.5 + 128).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def _frames_u8(out, image_mode):
    """[N, H, W, 3] uint8 frames of a generator output dict: out[image_mode], depth normalised per frame to [-1, 1] first."""
    img = out[image_mode]
    if image_mode == 'image_depth':                              # gen_videos_next3d.py:160-162, per frame
        img = -img
        lo, hi = img.amin(dim=(1, 2, 3), keepdim=True), img.amax(dim=(1, 2, 3), keepdim=True)
        img = (img - lo) / (hi - lo) * 2 - 1
        img = img.expand(-1, 3, -1, -1) if img.shape[1] == 1 else img
    return to_uint8_hwc(img)


def _depth_kw(image_mode, device):
    """Depth frames are clamped to their own depth range, as the scripts' one frame per call does (gen_videos_next3d.py:155,
    reenact_avatar_next3d.py:164), whatever the batching; the other image modes do not read the range.  The range is the CUDA
    renderer's (depth_range='image'); a generator on another device is called without the keyword."""
    return {'depth_range': 'image'} if image_mode == 'image_depth' and torch.device(device).type == 'cuda' else {}


def _frame_resolution(G, image_mode):
    return G.img_resolution if image_mode == 'image' else G.neural_rendering_resolution


def layout_cells(cells, gw, gh):
    """uint8 cells [F * gh * gw, h, w, C] (the cells of each frame in row-major grid order, frame after frame) -> frames
    [F, gh * h, gw * w, C]: layout_grid of gen_videos_next3d.py:35-49 per frame, on whatever device the cells are (the uint8
    conversion is per pixel, so converting the cells first and laying them out after gives the script's frames)."""
    n, h, w, C = cells.shape
    return cells.reshape(n // (gh * gw), gh, gw, h, w, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, gh * h, gw * w, C)


# ------------------------------------------------------------------------------------------------ plans and the two executors
class ShardPlan(NamedTuple):
    """How F frames are split into steps: rank r owns spans[r] and renders it in `steps` batches of `batch` frames; every rank runs
    the same number of steps (one collective each).  local_plan is the single-process run, shard_plan the sharded drivers'."""
    rank: int
    world: int
    spans: list
    batch: int
    steps: int

    def frames(self, k):
        """Global frame ids of this rank's batch k; a short tail repeats the last frame (one graph shape)."""
        a, b = self.spans[self.rank]
        lo = min(a + k * self.batch, max(b - 1, a))
        return [min(lo + j, b - 1) for j in range(self.batch)]

    def valid(self, k):
        """How many of frames(k) are this rank's own frames (the rest repeat the last)."""
        a, b = self.spans[self.rank]
        return max(0, min(self.batch, b - a - k * self.batch))

    def step_id(self, k):
        """Global id rank * steps + k of this rank's step k: the sampler seed offset of the step."""
        return self.rank * self.steps + k


def local_plan(F, batch):
    """The ShardPlan of a single process: F frames in ceil(F / batch) steps of exactly `batch` frames."""
    return ShardPlan(0, 1, [(0, F)], batch, -(-F // batch))


def shard_plan(F, batch):
    """The ShardPlan of F frames for this process's rank in the current torch.distributed world (world 1 when uninitialised).
    `batch` is an upper bound: the batch is the size in [batch/2, batch] that pads the largest rank's frame count least."""
    import torch.distributed as dist
    from . import distributed as D
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    spans = [D.shard_range(F, r, world) for r in range(world)]
    nmax = max(e - s for s, e in spans)
    batch = min(range(max(1, batch // 2), batch + 1), key=lambda bb: (-(-nmax // bb) * bb, -bb))     # least padding, then the largest
    return ShardPlan(rank, world, spans, batch, -(-nmax // batch))


class CallPlan(NamedTuple):
    """The calls of the single-process run local_plan(n, batch) that one rank makes to produce its own outputs [own[0], own[1]):
    every call whose window of items overlaps them, calls first .. first + steps - 1, each with the items, tail padding and step id
    (sampler seed offset) it has in the single-process run, so the outputs are those of that run whatever the number of ranks.
    A call that straddles the boundary of two ranks' outputs runs on both.  The step builders read it as a ShardPlan of one rank
    whose span is the window of its calls."""
    n: int
    batch: int
    own: tuple
    first: int
    steps: int
    rank = 0
    world = 1

    @property
    def spans(self):
        if self.steps == 0:
            return [self.own]
        return [(self.first * self.batch, min((self.first + self.steps) * self.batch, self.n))]

    def frames(self, k):
        """Item ids of call first + k: those of the single-process run, a short tail repeating item n - 1."""
        lo = (self.first + k) * self.batch
        return [min(lo + j, self.n - 1) for j in range(self.batch)]

    def step_id(self, k):
        return self.first + k

    def keep(self, k):
        """(lo, hi): the outputs frames(k)[lo:hi] are this rank's own."""
        lo = (self.first + k) * self.batch
        return max(self.own[0] - lo, 0), min(self.own[1] - lo, self.batch)


def call_plan(n, batch, own):
    """The CallPlan of the outputs own = (a, b) of n items in calls of `batch` (no calls when a >= b)."""
    a, b = own
    if a >= b:
        return CallPlan(n, batch, (a, b), 0, 0)
    return CallPlan(n, batch, (a, b), a // batch, (b - 1) // batch - a // batch + 1)


def head_plan(n_heads, batch, rank=0, world=1):
    """The CallPlan of `rank` of `world` over n_heads heads in calls of `batch` heads: whole calls, contiguous, in rank order
    (calls shard_range(ceil(n_heads / batch), r, world)), each with its single-process call index; no calls when a rank has none.
    Every call starts at one of the rank's own heads, so keep(k) is (0, n).  head_plan(n_heads, batch) makes the calls of
    local_plan(n_heads, batch)."""
    from . import distributed as D
    ca, cb = D.shard_range(-(-n_heads // batch), rank, world)
    return call_plan(n_heads, batch, (min(batch * ca, n_heads), min(batch * cb, n_heads)))


def gop_span(F, gop, rank, world):
    """Frames [a, b) of an F-frame video that `rank` of `world` renders and encodes: whole GOPs, contiguous, in rank order (rank r
    owns GOPs shard_range(ceil(F / gop), r, world)); empty when there are fewer GOPs than ranks."""
    from . import distributed as D
    a, b = D.shard_range(-(-F // gop), rank, world)
    return min(gop * a, F), min(gop * b, F)


def _sampler_kw(seed, sampler_noise, seed_id, ids):
    """Sampler keywords of one call: the rows ids (global image ids) of the per-image uniforms sampler_noise = (u_coarse [N, M, Dc, 1],
    u_fine [N, M, Df]) if given -- the renderer then draws no random numbers, so no seed goes with them --, else seed + seed_id (the
    global step id; 2 step and 2 step + 1 for the two calls of a multi-view head step, _head_views_step) if a seed is given, else
    none (a fresh random seed per call)."""
    if sampler_noise is not None:
        u_c, u_f = sampler_noise
        return {'sampler_noise': (u_c[ids], u_f[ids].reshape(-1, u_f.shape[-1]))}
    return {} if seed is None else {'seed': int(seed) + seed_id}


class _InOrder:
    """Items (meshes [1, V, 3], or (mesh, photo) pairs) of consecutive frames first, first + 1, ... from an in-order iterable, looked
    up by frame id as the batches advance (each id is read once; ids behind the current batch are dropped)."""

    def __init__(self, frames, first):
        self.it, self.next, self.have = iter(frames), first, {}

    def take(self, idx):
        while self.next <= max(idx):
            self.have[self.next] = next(self.it)
            self.next += 1
        self.have = {i: t for i, t in self.have.items() if i >= min(idx)}
        return [self.have[i] for i in idx]


def _in_order(plan, frames):
    """_InOrder over this rank's frames, frames(a, b) being an in-order iterable of the items of frames a .. b-1 (a rank without
    frames repeats the previous rank's last); None for a plan without steps."""
    if plan.steps == 0:
        return None
    first = plan.frames(0)[0]
    return _InOrder(frames(first, max(plan.spans[plan.rank][1], first + 1)), first)


def _steps(plan, step):
    """(step(k, plan.frames(k)), valid count) of every step of the plan, in order: the batches _to_host streams to the caller."""
    for k in range(plan.steps):
        yield step(k, plan.frames(k)), plan.valid(k)


def _to_host(batches, device):
    """uint8 numpy frames of successive batches of device frames (uint8 tensor [>= n, H, W, C], valid count n), in order; the
    device->host copy of batch i overlaps the work that produces batch i+1.  Each tensor must be fresh (not reused by its producer).
    A batch may also be a tuple of tensors [>= n, ...] of any dtype; then every item is the tuple of their rows."""
    cuda = torch.device(device).type == 'cuda'
    copy_s = torch.cuda.Stream(device) if cuda else None
    pending = None                                               # (host tensors, event, valid count, tuple batch) of the previous batch

    def drain(p):
        hosts, ev, n, many = p
        if ev is not None:
            ev.synchronize()
        for k in range(n):
            yield tuple(h[k].numpy() for h in hosts) if many else hosts[0][k].numpy()

    for dev_t, n in batches:
        many = isinstance(dev_t, tuple)
        ts = dev_t if many else (dev_t,)
        if cuda:
            hosts = tuple(torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in ts)
            copy_s.wait_stream(torch.cuda.current_stream(device))
            with torch.cuda.stream(copy_s):
                for host, t in zip(hosts, ts):
                    host.copy_(t, non_blocking=True)
                    t.record_stream(copy_s)
                ev = torch.cuda.Event()
                ev.record(copy_s)
        else:
            hosts, ev = ts, None
        if pending is not None:
            yield from drain(pending)
        pending = (hosts, ev, n, many)
    if pending is not None:
        yield from drain(pending)


def _gather_frames(plan, step, H, W, device, out):
    """The loop of the sharded drivers: for k in range(plan.steps), step(k, plan.frames(k)) renders this rank's batch k and returns
    its uint8 frames [plan.batch, H, W, 3]; they go to a ping-pong staging buffer, are gathered to rank 0 over NCCL on a side stream
    (world > 1) and copied to pinned host memory on a third stream, so the next batch renders while this one is in flight.
    -> [F, H, W, 3] uint8 host tensor on rank 0 (`out` if given), None elsewhere.  It is filled in stream order: the caller's
    current stream waits for the last copy, so synchronise that stream before reading the frames (back-to-back clips do not stall).
    A CPU `device` (host-side tests under gloo) runs the same loop without streams."""
    import contextlib
    import torch.distributed as dist
    rank, world, spans, batch = plan.rank, plan.world, plan.spans, plan.batch
    cuda = torch.device(device).type == 'cuda'
    host = None
    if rank == 0:
        host = out if out is not None else torch.empty(spans[-1][1], H, W, 3, dtype=torch.uint8, pin_memory=cuda)
    main = torch.cuda.current_stream(device) if cuda else None
    side, copy_s = (torch.cuda.Stream(device), torch.cuda.Stream(device)) if cuda else (None, None)

    def on(stream):
        return torch.cuda.stream(stream) if cuda else contextlib.nullcontext()

    def record(stream):
        if not cuda:
            return None
        ev = torch.cuda.Event()
        ev.record(stream)
        return ev
    stage = [torch.empty(batch, H, W, 3, dtype=torch.uint8, device=device) for _ in range(2)]
    gath = [torch.empty(world, batch, H, W, 3, dtype=torch.uint8, device=device) if rank == 0 and world > 1 else None for _ in range(2)]
    drained = [None, None]
    for k in range(plan.steps):
        frames = step(k, plan.frames(k))
        s = k & 1
        if drained[s] is not None:
            main.wait_event(drained[s])                                    # batch k-2 has left this staging buffer
        stage[s].copy_(frames)
        if cuda:
            side.wait_stream(main)
        with on(side):
            if world > 1:
                dist.gather(stage[s], list(gath[s].unbind(0)) if rank == 0 else None, dst=0)
            ev = record(side)
        drained[s] = ev
        if rank == 0:
            if cuda:
                copy_s.wait_event(ev)
            with on(copy_s):
                for r in range(world):
                    s0, e0 = spans[r]
                    f0 = s0 + k * batch
                    n = max(0, min(batch, e0 - f0))
                    if n > 0:
                        src = gath[s][r] if world > 1 else stage[s]
                        host[f0:f0 + n].copy_(src[:n], non_blocking=cuda)
                ev2 = record(copy_s)
            drained[s] = ev2                                               # the staging / gather buffers are free once the D2H left them
    if cuda:
        main.wait_stream(side)
        main.wait_stream(copy_s)
    return host


def _own_frames(plan, step, grid=None):
    """uint8 device frames [n, H, W, 3] of this rank's own outputs, batch after batch: step(k, plan.frames(k)) for each call of the
    CallPlan, trimmed to plan.keep(k).  grid = (gw, gh): the items are the cells of frames, laid out (_whole_frames) from the rank's
    first own cell to its last."""
    def own():
        for k in range(plan.steps):
            lo, hi = plan.keep(k)
            yield step(k, plan.frames(k))[lo:], hi - lo
    for u8, n in (own() if grid is None else _whole_frames(own(), *grid)):
        yield u8[:n]


def write_video_sharded(path, shard, encoder, group=None):
    """The per-rank loop of a video split over the ranks of `group` (gloo; None = the default group, or one process when
    torch.distributed is not initialised).  shard() -> ((a, b), frames): this rank's frames [a, b) (gop_span; possibly none) and an
    iterable of their uint8 device frame batches in order (the *_video_shard drivers); encoder(width, height, a) -> an encoder of
    frames a, a + 1, ... (video.H264Encoder: write(frames) / flush() -> [(sample, is_idr)], width, height, fps, sps, pps).  The
    frames go straight from the renderer to the encoder on the device, and only the coded samples leave it: they are gathered to
    rank 0 over `group` on host memory, and rank 0 writes them, in frame order, to one MP4 at `path` (none when there are no
    frames).  A failure on any rank -- its rank and message -- reaches every rank at the gather, which then raises
    distributed.RankError on every rank, and no file is left behind; in one process the exception propagates as it is."""
    from . import distributed as D, mp4
    rank, world = D.rank_world(group)
    err, payload = None, None
    try:
        (a, b), frames = shard()
        enc, samples = None, []
        for f in frames:
            if enc is None:
                enc = encoder(f.shape[2], f.shape[1], a)
            samples += enc.write(f)
        if enc is not None:
            samples += enc.flush()
        if len(samples) != b - a:
            raise RuntimeError(f'frames {a}..{b - 1}: {len(samples)} coded frames')
        payload = (samples, None if enc is None else (enc.width, enc.height, enc.fps, enc.sps, enc.pps))
    except Exception as e:
        if world == 1:
            raise
        err = f'{type(e).__name__}: {e}'
    D.agree(err, group)
    parts = D.gather_to_root(payload, group)
    err = None
    if rank == 0:
        try:
            heads = {h for _, h in parts if h is not None}
            if len(heads) > 1:
                raise RuntimeError('the ranks coded different parameter sets')
            if heads:
                with mp4.Mp4Writer(path, *heads.pop()) as w:
                    for samples, _ in parts:
                        for sample, idr in samples:
                            w.add(sample, idr)
        except Exception as e:
            import os
            if os.path.exists(path):
                os.remove(path)
            if world == 1:
                raise
            err = f'{type(e).__name__}: {e}'
    D.agree(err, group)


# ------------------------------------------------------------------------------------------------ frames and orbits (gen_videos_next3d.py)
def render_frames(G, ws_frames, cams, verts, batch=8, image_mode='image', noise_mode='const', device=None, seed=None, sampler_noise=None):
    """Yield one uint8 HWC numpy frame per (ws, camera, mesh) triple, in order, rendering `batch` frames per synthesis call.

    ws_frames [F, L, D], cams [F, 25], verts: [F, V, 3] / [1, V, 3] (static mesh) tensors, or an iterable of per-frame [1, V, 3]
    tensors (e.g. inputs.FramePrefetcher).  The last, partial batch is padded by repeating its final frame (one graph shape) and
    the padding is dropped.  The device->host copy of batch i overlaps the synthesis of batch i+1.  `seed`: base seed of the ray
    sampler's RNG (batch k uses seed + k); None = a fresh random seed per call, like the reference's torch.rand.
    `sampler_noise=(u_coarse [F, M, Dc, 1], u_fine [F, M, Df])`: per-frame sampler uniforms instead of the in-kernel RNG and `seed`
    (parity tests: frame f gets the same noise whichever batch slot it lands in).  image_mode 'image_depth' renders with
    depth_range='image', so each depth frame is clamped to its own range as in the script (one frame per synthesis call), whatever
    the batching."""
    device = device or next(G.parameters()).device
    plan = local_plan(ws_frames.shape[0], batch)
    verts = verts if torch.is_tensor(verts) else _InOrder(verts, 0)
    yield from _to_host(_steps(plan, _frames_step(G, plan, ws_frames, cams, verts, image_mode, noise_mode, device, seed,
                                                  sampler_noise)), device)


def render_frames_sharded(G, ws_frames, cams, verts, batch=8, noise_mode='const', seed=0, device=None, out=None, sampler_noise=None):
    """Strong-scaling video driver (BASELINE.json configs[3]: one clip split over the GPUs of a box): rank r renders the contiguous
    frame range shard_range(F, r, world) in batches through `G.synthesis`, converts to uint8 HWC on the device (4x fewer bytes than
    the fp32 images) and the batches are gathered to rank 0 over NCCL on a side stream from a ping-pong staging buffer, so batch
    i+1 renders while batch i is in flight; rank 0 copies every gathered batch to pinned host memory on a third stream.
    Returns the [F, H, W, 3] uint8 host tensor (frame order) on rank 0, None elsewhere, filled in stream order (synchronise the
    current stream before reading it).  World size 1: no collective.
    `batch` is an upper bound: the per-call batch is the size in [batch/2, batch] that pads the rank's frame count least (30 frames per
    rank -> 5 batches of 6, not 4 of 8).  `out`: optional pinned [F, H, W, 3] uint8 host tensor to fill on rank 0 (pinning 190 MB per
    clip costs tens of milliseconds).  `sampler_noise`: per-frame uniforms as in render_frames, rows indexed by the global frame id,
    so the frames do not depend on the number of ranks (batch k of rank r otherwise draws sampler seed seed + r * steps + k)."""
    device = device or next(G.parameters()).device
    plan = shard_plan(ws_frames.shape[0], batch)
    step = _frames_step(G, plan, ws_frames, cams, verts, 'image', noise_mode, device, seed, sampler_noise)
    return _gather_frames(plan, step, G.img_resolution, G.img_resolution, device, out)


def _frames_step(G, plan, ws, cams, verts, image_mode, noise_mode, device, seed, sampler_noise, reuse_backbone=False):
    """step(k, idx) of the frame and reenactment drivers: the uint8 frames of the frames idx, one synthesis call.  ws: per-frame
    latents [F, L, D], or [1, L, D] for one identity; verts: per-frame [F, V, 3] or static [1, V, 3] meshes, or an _InOrder source of
    [1, V, 3] meshes.  reuse_backbone: every frame has the same ws (one identity), so the first step caches the ws-only backbones and
    the later ones reuse them (use_cached_backbone); with noise_mode 'const' or 'none' those are a function of ws alone, so the frames
    are the same."""
    def rows(t, idx):
        if t.shape[0] == 1:
            return t.to(device, torch.float32).expand(len(idx), -1, -1)
        return t[idx].to(device, torch.float32, non_blocking=True)

    def step(k, idx):
        w = rows(ws, idx)
        c = cams[idx].to(device, torch.float32, non_blocking=True)
        v = torch.cat(verts.take(idx), 0).to(device, torch.float32, non_blocking=True) if isinstance(verts, _InOrder) else rows(verts, idx)
        kw = _sampler_kw(seed, sampler_noise, plan.step_id(k), idx)
        if reuse_backbone:
            kw['use_cached_backbone' if k else 'cache_backbone'] = True
        return _frames_u8(G.synthesis(w, c, v, noise_mode=noise_mode, **_depth_kw(image_mode, device), **kw), image_mode)
    return step


def render_orbit(G, ws, cams, verts, batch=8, image_mode='image', seed=None, sampler_noise=None):
    """Yield one uint8 HWC numpy frame per camera of cams [F, 25] for ONE head: ws [1, L, D] and mesh verts [1, V, 3] stay fixed
    (gen_videos_next3d.py with one seed, sample sheets), so the tri-planes are computed once (noise_mode 'const') and every batch of
    `batch` cameras is rendered from them by G.render_views -- volume rendering and super-resolution only.  Padding, `seed` and
    `sampler_noise` as in render_frames."""
    device = next(G.parameters()).device
    plan = local_plan(cams.shape[0], batch)
    yield from _to_host(_steps(plan, _orbit_step(G, plan, ws, cams, verts, image_mode, device, seed, sampler_noise)), device)


def render_orbit_sharded(G, ws, cams, verts, batch=8, image_mode='image', seed=0, sampler_noise=None, out=None, device=None):
    """render_orbit over the GPUs of a box: every rank computes the head's planes once (ws [1, L, D], mesh verts [1, V, 3]) and
    renders its contiguous range of the cameras cams [F, 25] with G.render_views; the frames are gathered to rank 0 as in
    render_frames_sharded.  -> [F, H, W, 3] uint8 host tensor on rank 0, None elsewhere.  `sampler_noise` rows are indexed by the
    global frame id."""
    device = device or next(G.parameters()).device
    plan = shard_plan(cams.shape[0], batch)
    step = _orbit_step(G, plan, ws, cams, verts, image_mode, device, seed, sampler_noise)
    res = _frame_resolution(G, image_mode)
    return _gather_frames(plan, step, res, res, device, out)


def orbit_video_shard(G, ws, cams, verts, gop, rank=0, world=1, batch=8, image_mode='image', seed=None):
    """render_orbit's video split over ranks for write_video_sharded: -> ((a, b), frames), this rank's frames [a, b) =
    gop_span(F, gop, rank, world) as uint8 device frame batches, from exactly the render_views calls of render_orbit that hold
    them (CallPlan), so the frames are render_orbit's.  A rank without frames computes nothing."""
    device = next(G.parameters()).device
    span = gop_span(cams.shape[0], gop, rank, world)
    plan = call_plan(cams.shape[0], batch, span)
    if plan.steps == 0:
        return span, iter(())
    return span, _own_frames(plan, _orbit_step(G, plan, ws, cams, verts, image_mode, device, seed, None))


def _orbit_step(G, plan, ws, cams, verts, image_mode, device, seed, sampler_noise):
    """Computes and caches the head's tri-planes; -> step(k, idx): the uint8 frames of the cameras idx, one render_views call."""
    G.synthesis(ws.to(device, torch.float32), cams[:1].to(device, torch.float32), verts.to(device, torch.float32), noise_mode='const',
                cache_backbone=True, seed=0)

    def step(k, idx):
        out = G.render_views(cams[idx].to(device, torch.float32, non_blocking=True), **_depth_kw(image_mode, device),
                             **_sampler_kw(seed, sampler_noise, plan.step_id(k), idx))
        return _frames_u8(out, image_mode)
    return step


# ------------------------------------------------------------------------------------------------ reenactment (reenact_avatar_next3d.py)
def reenact_schedule(drive_root, num_frames, lms_cond=True):
    """Frame schedule of reenact_avatar_next3d.py:125-160 for a driving directory (dataset.json + NNN.png / NNN.obj / NNN_kpt2d.txt):
    the script walks the sorted PNG list, skips k = 0, stops after k = num_frames and smooths the camera over the labels k-1, k, k+1
    (so the last usable frame is len(labels) - 2; the script itself runs into an IndexError there).
    -> dict(ks, ids, png_paths, obj_paths, lms_paths (or None), cams float32 [F, 25])."""
    import glob
    import os
    from . import inputs
    labels = inputs.load_labels(os.path.join(drive_root, 'dataset.json'))
    img_list = sorted(glob.glob(drive_root + '/*.png'))
    ks = [k for k in range(len(img_list)) if 1 <= k <= num_frames and k + 1 < len(labels)]
    ids = [os.path.basename(img_list[k]).split('.')[0] for k in ks]
    return dict(ks=ks, ids=ids, png_paths=[img_list[k] for k in ks], obj_paths=[drive_root + f'/{i}.obj' for i in ids],
                lms_paths=[drive_root + f'/{i}_kpt2d.txt' for i in ids] if lms_cond else None,
                cams=inputs.smoothed_cameras(labels, ks))


def reenact_frames(G, ws, drive_root, num_frames, batch=8, lms_cond=True, fixed_camera=None, noise_mode='const', seed=None,
                   sampler_noise=None, prefetch_depth=8, workers=4, image_mode='image'):
    """reenact_avatar_next3d.py:125-167 for ONE identity `ws` [1, L, D]: yields the rendered uint8 HWC frame of every driving frame,
    in order.  Meshes are parsed by the native parsers on worker threads (inputs.FramePrefetcher, pinned memory) while the GPU renders
    batches of `batch` frames; `fixed_camera` [1, 25] replaces the per-frame cameras (the script's --fixed_camera).
    A `.n3dpack` file written by inputs.write_frame_pack can be given instead of a directory (no parsing at all).  image_mode as in
    render_frames; for noise_mode 'const' / 'none' the first batch caches the ws-only backbones and the later ones reuse them."""
    n, cams, frames = _reenact_source(drive_root, num_frames, lms_cond, fixed_camera, prefetch_depth, workers)
    device = next(G.parameters()).device
    plan = local_plan(n, batch)
    yield from _to_host(_steps(plan, _reenact_step(G, plan, ws, cams, frames, image_mode, noise_mode, device, seed, sampler_noise)),
                        device)


def reenact_frames_sharded(G, ws, drive_root, num_frames, batch=8, lms_cond=True, fixed_camera=None, noise_mode='const', seed=0,
                           sampler_noise=None, image_mode='image', out=None, device=None, prefetch_depth=8, workers=4):
    """reenact_frames over the GPUs of a box (one process per GPU, as render_frames_sharded): every rank computes the frame schedule
    (reenact_schedule, or the pack's cameras), parses -- or reads from the memory-mapped `.n3dpack` -- only the meshes of its own
    contiguous frame range, and renders them in batches; for noise_mode 'const' / 'none' its first batch caches the ws-only backbones
    and the later ones reuse them.  The uint8 frames are gathered to rank 0 as in render_frames_sharded.
    -> [F, H, W, 3] uint8 host tensor on rank 0 (F = the schedule's frame count; H = W = G.img_resolution for 'image', the neural
    rendering resolution for 'image_raw' / 'image_depth'), None elsewhere.  `sampler_noise` rows are indexed by the global frame id;
    image_mode and `batch` as in reenact_frames / render_frames_sharded."""
    device = device or next(G.parameters()).device
    n, cams, frames = _reenact_source(drive_root, num_frames, lms_cond, fixed_camera, prefetch_depth, workers)
    plan = shard_plan(n, batch)
    step = _reenact_step(G, plan, ws, cams, frames, image_mode, noise_mode, device, seed, sampler_noise)
    res = _frame_resolution(G, image_mode)
    return _gather_frames(plan, step, res, res, device, out)


def _reenact_step(G, plan, ws, cams, frames, image_mode, noise_mode, device, seed, sampler_noise):
    """step(k, idx) of the reenactment drivers: _frames_step of the identity ws with the meshes of this rank's driving frames."""
    ws = ws.detach().to(device, torch.float32).reshape(1, *ws.shape[-2:])
    return _frames_step(G, plan, ws, cams, _in_order(plan, frames), image_mode, noise_mode, device, seed, sampler_noise,
                        noise_mode in ('const', 'none'))


def _reenact_source(drive_root, num_frames, lms_cond, fixed_camera, prefetch_depth, workers, photos=False):
    """(frame count n, cameras [n, 25], frames(a, b) -> in-order iterable of the [1, V, 3] meshes of frames a .. b-1) of a driving
    directory (reenact_schedule; only the requested frames are parsed, on worker threads) or of a `.n3dpack` (memory-mapped).
    photos=True: frames(a, b) yields (mesh, uint8 photo [512, 512, 3]) pairs (a directory only: a pack carries no photos)."""
    from . import inputs
    if str(drive_root).endswith('.n3dpack'):
        if photos:
            raise ValueError(f'{drive_root}: a .n3dpack carries no driving photos; pass the driving directory')
        pack = inputs.FramePack(drive_root)
        n = min(len(pack), num_frames)
        cams = torch.from_numpy(np.array(pack.cams[:n]))

        def frames(a, b):
            return pack[a:b]
    else:
        sch = reenact_schedule(drive_root, num_frames, lms_cond)
        n = len(sch['ks'])
        cams = sch['cams']
        pairs = list(zip(sch['obj_paths'], sch['lms_paths'] if lms_cond else [None] * n))

        def frames(a, b):
            return inputs.FramePrefetcher(pairs[a:b], depth=prefetch_depth, workers=workers,
                                          photos=sch['png_paths'][a:b] if photos else None)
    if fixed_camera is not None:
        cams = fixed_camera.reshape(1, 25).cpu().float().expand(n, -1)
    return n, cams, frames


def interpolate_ws_device(ws_keyframes, w_frames, wraps=2, kind='cubic'):
    """interpolate_ws on the device: the spline is linear in its knots, so its basis B [K * w_frames, K] (interp1d evaluated once on
    the identity, wrap-around tiling folded in) is built on the host and the frames are B @ ws_keyframes in one small kernel
    (n3d_interp_rows) -- the latents never visit the host.  float32; equals interpolate_ws to ~1e-6."""
    from . import kernels as K
    B = interpolation_basis(ws_keyframes.shape[0], w_frames, wraps, kind).to(ws_keyframes.device, torch.float32).contiguous()
    return K.interp_rows(B, ws_keyframes.to(torch.float32).contiguous())


def interpolation_basis(Kf, w_frames, wraps=2, kind='cubic'):
    """The float64 basis [Kf * w_frames, Kf] of interpolate_ws over Kf keyframes: frame f is sum_k B[f, k] * keyframe k."""
    import scipy.interpolate
    x = np.arange(-Kf * wraps, Kf * (wraps + 1))
    eye = np.tile(np.eye(Kf), [wraps * 2 + 1, 1])                                  # knot i of the tiled sequence is keyframe i % K
    return torch.from_numpy(scipy.interpolate.interp1d(x, eye, kind=kind, axis=0)(np.arange(Kf * w_frames) / w_frames))


# ------------------------------------------------------------------------------------------------ grids (--grid of both scripts)
def _grid_seeds(seeds, grid, num_keyframes, shuffle_seed):
    """(seed of every keyframe of every cell [K * gh * gw] int64, K): gen_videos_next3d.py:78-92."""
    gw, gh = grid
    if num_keyframes is None:
        if len(seeds) % (gw * gh) != 0:
            raise ValueError('Number of input seeds must be divisible by grid W*H')
        num_keyframes = len(seeds) // (gw * gh)
    all_seeds = np.zeros(num_keyframes * gh * gw, dtype=np.int64)
    for idx in range(num_keyframes * gh * gw):
        all_seeds[idx] = seeds[idx % len(seeds)]
    if shuffle_seed is not None:
        np.random.RandomState(seed=shuffle_seed).shuffle(all_seeds)
    return all_seeds, num_keyframes


def _frontal_camera(G, n):
    """c [n, 25]: the frontal conditioning camera of gen_videos_next3d.py:96-100 (avg_camera_pivot / avg_camera_radius, focal 4.2647)."""
    rk = G.rendering_kwargs
    pose = camera.look_at_pose(3.14 / 2, 3.14 / 2, torch.tensor(rk['avg_camera_pivot']), rk['avg_camera_radius'])
    intr = torch.tensor([[FOCAL_FFHQ, 0, 0.5], [0, FOCAL_FFHQ, 0.5], [0, 0, 1]], dtype=torch.float32)
    return torch.cat([pose.reshape(-1, 16), intr.reshape(-1, 9)], 1).repeat(n, 1)


def grid_keyframes(G, seeds, grid, num_keyframes=None, shuffle_seed=None, truncation_psi=1, truncation_cutoff=14):
    """The keyframe latents of an interpolation grid video (gen_videos_next3d.py:78-106, `--grid=WxH`): grid = (gw, gh); seeds repeat
    as seeds[idx % len(seeds)] over K * gh * gw keyframes (K = num_keyframes, else len(seeds) / (gw * gh), which must divide: ValueError
    otherwise), optionally shuffled by RandomState(shuffle_seed); z = RandomState(seed).randn(z_dim), mapped with the frontal camera.
    -> ws [gh, gw, K, L, D] on the generator's device."""
    gw, gh = grid
    all_seeds, K = _grid_seeds(seeds, grid, num_keyframes, shuffle_seed)
    device = next(G.parameters()).device
    zs = seed_latents(all_seeds, G.z_dim).to(device)
    ws = G.mapping(z=zs, c=_frontal_camera(G, len(zs)).to(device), truncation_psi=truncation_psi, truncation_cutoff=truncation_cutoff)
    return ws.reshape(gh, gw, K, *ws.shape[1:])


def _whole_frames(cell_batches, gw, gh):
    """(uint8 frames [nf, gh * h, gw * w, 3], nf) from successive batches (uint8 cells [>= n, h, w, 3], valid count n) of a cell
    sequence ordered frame-major, cell-minor: a frame is laid out as soon as its last cell has been rendered."""
    per, rest = gw * gh, None
    for u8, n in cell_batches:
        cur = u8[:n] if rest is None else torch.cat([rest, u8[:n]])
        nf = cur.shape[0] // per
        rest = cur[nf * per:]
        if nf:
            yield layout_cells(cur[:nf * per], gw, gh), nf


def render_grid_frames(G, ws_grid, verts, w_frames, batch=8, image_mode='image', seed=None, sampler_noise=None):
    """gen_videos_next3d.py:77-171 with `--grid=WxH`: yield one uint8 HWC numpy frame [gh * R, gw * R, 3] per frame of the video
    (F = K * w_frames frames for ws_grid [gh, gw, K, L, D] from grid_keyframes), laid out like the script's layout_grid.  Cell
    (yi, xi) interpolates its own keyframes; all cells of a frame share its orbit camera and the static mesh verts [1, V, 3]
    (noise_mode 'const').  The F * gh * gw images run frame-major, cell-minor through `synthesis` in batches of `batch` (the last
    one padded as in render_frames), so a batch may hold parts of two frames.  'image_depth' cells are normalised and clamped per
    cell, as the script's one image per call; the frames stay 3-channel (the script writes 1-channel depth frames).  `seed` as in
    render_frames; `sampler_noise=(u_coarse [F * cells, M, Dc, 1], u_fine [F * cells, M, Df])` rows are indexed by the global
    image id f * gh * gw + yi * gw + xi."""
    device = next(G.parameters()).device
    gh, gw, K = ws_grid.shape[:3]
    plan = local_plan(K * w_frames * gh * gw, batch)                                # batches of images
    step = _grid_step(G, plan, ws_grid, verts, w_frames, image_mode, device, seed, sampler_noise)
    yield from _to_host(_whole_frames(_steps(plan, step), gw, gh), device)


def render_grid_frames_sharded(G, ws_grid, verts, w_frames, batch=8, image_mode='image', seed=0, sampler_noise=None, out=None,
                               device=None):
    """render_grid_frames over the GPUs of a box (one process per GPU, as render_frames_sharded), sharded by frame: all cells of a
    frame render on one rank, plan.batch frames (batch // cells as the bound, at least 1) of gh * gw cells per synthesis call.
    -> [F, gh * R, gw * R, 3] uint8 host tensor on rank 0, None elsewhere.  `sampler_noise` rows are indexed by the global image id
    f * gh * gw + cell, so the frames do not depend on the number of ranks."""
    device = device or next(G.parameters()).device
    gh, gw, K = ws_grid.shape[:3]
    cells = gh * gw
    plan = shard_plan(K * w_frames, max(1, batch // cells))                        # batches of frames
    images = _grid_step(G, plan, ws_grid, verts, w_frames, image_mode, device, seed, sampler_noise)

    def step(k, idx):
        return layout_cells(images(k, [f * cells + j for f in idx for j in range(cells)]), gw, gh)
    res = _frame_resolution(G, image_mode)
    return _gather_frames(plan, step, gh * res, gw * res, device, out)


def grid_video_shard(G, ws_grid, verts, w_frames, gop, rank=0, world=1, batch=8, image_mode='image', seed=None):
    """render_grid_frames's video split over ranks for write_video_sharded: -> ((a, b), frames), this rank's frames [a, b) =
    gop_span(F, gop, rank, world) as uint8 device frame batches.  The items are images, as in render_grid_frames: the rank makes
    exactly the synthesis calls of render_grid_frames that hold one of its images (same images, padding and seed), keeps its own
    images and lays them out from its first frame, so the frames are render_grid_frames's."""
    device = next(G.parameters()).device
    gh, gw, K = ws_grid.shape[:3]
    cells = gh * gw
    a, b = gop_span(K * w_frames, gop, rank, world)
    plan = call_plan(K * w_frames * cells, batch, (a * cells, b * cells))
    if plan.steps == 0:
        return (a, b), iter(())
    return (a, b), _own_frames(plan, _grid_step(G, plan, ws_grid, verts, w_frames, image_mode, device, seed, None), (gw, gh))


def _grid_step(G, plan, ws_grid, verts, w_frames, image_mode, device, seed, sampler_noise):
    """The schedule of a grid video, image f * cells + cell: every cell interpolates its own keyframes (interpolate_ws_device: cubic,
    2 wraps), every cell of frame f has the frame's orbit camera (gen_videos_next3d.py:128-144).  -> step(k, ids): the uint8 cells
    [len(ids), R, R, 3] of the global image ids, one synthesis call."""
    gh, gw, K = ws_grid.shape[:3]
    F = K * w_frames
    wsf = torch.stack([interpolate_ws_device(ws_grid[yi, xi].to(device), w_frames) for yi in range(gh) for xi in range(gw)], 1)
    wsf = wsf.reshape(F * gh * gw, *wsf.shape[2:])
    rk = G.rendering_kwargs
    cams = orbit_camera_params(F, torch.tensor(rk['avg_camera_pivot']), rk['avg_camera_radius']).repeat_interleave(gh * gw, 0)
    v = verts.to(device, torch.float32).reshape(1, *verts.shape[-2:])

    def step(k, ids):
        out = G.synthesis(wsf[ids], cams[ids].to(device, torch.float32, non_blocking=True), v.expand(len(ids), -1, -1),
                          noise_mode='const', **_depth_kw(image_mode, device), **_sampler_kw(seed, sampler_noise, plan.step_id(k), ids))
        return _frames_u8(out, image_mode)
    return step


def photo_cell(photo, device):
    """uint8 driving photo [H, W, 3] -> its uint8 grid cell [H, W, 3] through the script's float32 arithmetic on `device`:
    `/ 127.5 - 1` (reenact_avatar_next3d.py:134-135), then layout_grid's conversion."""
    img = photo.to(device, non_blocking=True).permute(2, 0, 1).float().unsqueeze(0) / 127.5 - 1.
    return to_uint8_hwc(img)[0]


def _check_reenact_grid(G, S, grid):
    gw, gh = grid
    if gw * gh != S + 1:
        raise ValueError(f'grid {gw}x{gh} has {gw * gh} cells, but the driving photo and {S} avatar(s) need {S + 1}')
    if G.img_resolution != 512:
        raise ValueError(f'a reenactment grid needs img_resolution 512 (the photo cell is a 512x512 crop), got {G.img_resolution}')


def reenact_grid_frames(G, ws, drive_root, num_frames, grid, batch=8, lms_cond=True, fixed_camera=None, noise_mode='const', seed=None,
                        sampler_noise=None, prefetch_depth=8, workers=4):
    """reenact_avatar_next3d.py:116-167 with several seeds and `--grid=WxH`: one mesh drives S identities ws [S, L, D]; every frame is
    the grid (gw, gh) = grid of the driving photo followed by the S avatars (gw * gh must be S + 1, else ValueError), yielded as a
    uint8 HWC numpy frame [gh * 512, gw * 512, 3] equal to the script's layout_grid.  'image' output at img_resolution 512 only.
    The photo is the PNG's 512x512 crop, decoded on the prefetcher's worker threads next to the mesh (a `.n3dpack` carries no photos:
    ValueError).  Each synthesis call renders S heads x k frames (k = max(1, batch // S), the last batch padded), head-major; with
    noise_mode 'const' / 'none' the S heads' ws-only backbones are computed once and every batch reuses them (use_cached_backbone),
    with 'random' every batch runs the full path.  `seed`: batch b draws sampler seed seed + b; `sampler_noise=(u_coarse
    [F * S, M, Dc, 1], u_fine [F * S, M, Df])` rows are indexed f * S + s (frame f, identity s)."""
    _check_reenact_grid(G, ws.shape[0], grid)
    n, cams, frames = _reenact_source(drive_root, num_frames, lms_cond, fixed_camera, prefetch_depth, workers, photos=True)
    device = next(G.parameters()).device
    plan = local_plan(n, max(1, batch // ws.shape[0]))
    step = _reenact_grid_step(G, plan, ws, cams, frames, grid, noise_mode, device, seed, sampler_noise)
    yield from _to_host(_steps(plan, step), device)


def reenact_grid_frames_sharded(G, ws, drive_root, num_frames, grid, batch=8, lms_cond=True, fixed_camera=None, noise_mode='const',
                                seed=0, sampler_noise=None, out=None, device=None, prefetch_depth=8, workers=4):
    """reenact_grid_frames over the GPUs of a box, sharded by frame as reenact_frames_sharded (each rank parses the meshes and decodes
    the photos of its own frames only; plan.batch frames of S heads per call, batch // S as the bound).  -> [F, gh * 512, gw * 512, 3]
    uint8 host tensor on rank 0, None elsewhere.  `sampler_noise` rows are indexed f * S + s by the global frame id f."""
    _check_reenact_grid(G, ws.shape[0], grid)
    device = device or next(G.parameters()).device
    n, cams, frames = _reenact_source(drive_root, num_frames, lms_cond, fixed_camera, prefetch_depth, workers, photos=True)
    plan = shard_plan(n, max(1, batch // ws.shape[0]))
    step = _reenact_grid_step(G, plan, ws, cams, frames, grid, noise_mode, device, seed, sampler_noise)
    gw, gh = grid
    return _gather_frames(plan, step, gh * 512, gw * 512, device, out)


def reenact_grid_video_shard(G, ws, drive_root, num_frames, grid, gop, rank=0, world=1, batch=8, lms_cond=True, fixed_camera=None,
                             noise_mode='const', seed=None, prefetch_depth=8, workers=4):
    """reenact_grid_frames's video split over ranks for write_video_sharded: -> ((a, b), frames), this rank's frames [a, b) =
    gop_span(F, gop, rank, world) as uint8 device frame batches.  The items are driving frames of S heads: the rank makes exactly
    the calls of reenact_grid_frames that hold one of its frames, parsing only their meshes and photos; with noise_mode 'const' /
    'none' its own first call caches the ws-only backbones, which are then those of the single-process run."""
    _check_reenact_grid(G, ws.shape[0], grid)
    n, cams, frames = _reenact_source(drive_root, num_frames, lms_cond, fixed_camera, prefetch_depth, workers, photos=True)
    device = next(G.parameters()).device
    span = gop_span(n, gop, rank, world)
    plan = call_plan(n, max(1, batch // ws.shape[0]), span)
    if plan.steps == 0:
        return span, iter(())
    return span, _own_frames(plan, _reenact_grid_step(G, plan, ws, cams, frames, grid, noise_mode, device, seed, None))


def _reenact_grid_step(G, plan, ws, cams, frames, grid, noise_mode, device, seed, sampler_noise):
    """step(k, idx): the uint8 grid frames [len(idx), gh * 512, gw * 512, 3] of the driving frames idx.  One synthesis call renders
    the S heads x len(idx) frames, head-major (image n is head n // len(idx)); noise_mode 'const' / 'none': the S heads' ws-only
    backbones come from the engine's cache, filled by the first step."""
    S = ws.shape[0]
    wsd = ws.detach().to(device, torch.float32).reshape(S, *ws.shape[-2:])
    wsb = wsd.repeat_interleave(plan.batch, 0)
    src = _in_order(plan, frames)

    def step(k, idx):
        items = src.take(idx)                                                      # (mesh [1, V, 3], photo) pairs
        c = cams[idx].to(device, torch.float32, non_blocking=True)
        v = torch.cat([mesh for mesh, _ in items], 0).to(device, torch.float32, non_blocking=True)
        kw = _sampler_kw(seed, sampler_noise, plan.step_id(k), [f * S + s for s in range(S) for f in idx])
        if noise_mode in ('const', 'none'):
            if k == 0:
                G.synthesis(wsd, c[:1].expand(S, -1), v[:1].expand(S, -1, -1), noise_mode=noise_mode, cache_backbone=True, seed=0)
            kw['use_cached_backbone'] = True
        av = _frames_u8(G.synthesis(wsb, c.repeat(S, 1), v.repeat(S, 1, 1), noise_mode=noise_mode, **kw), 'image')
        av = av.reshape(S, len(idx), *av.shape[1:]).transpose(0, 1)                   # [len(idx), S, H, W, 3]
        photos = torch.stack([photo_cell(p, device) for _, p in items])[:, None]
        cells = torch.cat([photos, av], 1)
        return layout_cells(cells.reshape(-1, *cells.shape[2:]), *grid)
    return step


# ------------------------------------------------------------------------------------------------ shape extraction (row f2)
def create_samples(N, cube_length, head=0, count=None, device='cpu'):
    """Voxel-grid query points [1, count, 3] of `create_samples` (gen_samples_next3d.py:80-102) for the flat indices
    head .. head+count-1, computed with the reference's own float32 operations (including its float -- not floor -- division,
    which shears the y / x columns by idx / N, and the float32 rounding of indices above 2^24), so that any chunk is bit-identical
    to the corresponding slice of the reference's full N^3 tensor without materialising it (201 MB at N = 256, 1.6 GB at 512)."""
    count = N ** 3 - head if count is None else count
    voxel_origin = np.array([0, 0, 0]) - cube_length / 2
    voxel_size = cube_length / (N - 1)
    idx = torch.arange(head, head + count, dtype=torch.int64, device=device)
    s = torch.zeros(count, 3, device=device)
    s[:, 2] = idx % N
    s[:, 1] = (idx.float() / N) % N
    s[:, 0] = ((idx.float() / N) / N) % N
    s[:, 0] = (s[:, 0] * voxel_size) + voxel_origin[2]
    s[:, 1] = (s[:, 1] * voxel_size) + voxel_origin[1]
    s[:, 2] = (s[:, 2] * voxel_size) + voxel_origin[0]
    return s.unsqueeze(0)


def trim_sigma_grid(sigmas, shape_res, pad_value=-1000.0):
    """flip + border trim of gen_samples_next3d.py:226-238 on a [R,R,R] tensor (device or host)."""
    sigmas = torch.flip(sigmas, dims=[0])
    pad = int(30 * shape_res / 256)
    for d in range(3):
        sl = [slice(None)] * 3
        sl[d] = slice(0, pad)
        sigmas[tuple(sl)] = pad_value
        sl[d] = slice(shape_res - pad, shape_res)
        sigmas[tuple(sl)] = pad_value
    return sigmas


def _sigma_grid(G, ws, v, shape_res, noise_mode):
    """The density grid of extract_sigma_grid, as a float32 CUDA tensor [R, R, R]."""
    from . import kernels as K
    eng = G._get_engine()
    eng.rk = G.rendering_kwargs
    planes = eng.compute_planes(ws, v, noise_mode)
    box = G.rendering_kwargs['box_warp']
    sigmas = torch.empty(shape_res, shape_res, shape_res, device=planes.device)
    # one launch: voxel centres generated in the kernel (bit-identical to create_samples), flip + border trim fused into the store,
    # border voxels (55 % of a 256^3 grid) never decoded
    K.sample_grid(planes[0], shape_res, box * 1, box, eng.dec, sigmas, pad=int(30 * shape_res / 256))
    return sigmas


def extract_sigma_grid(G, ws, v, shape_res=512, max_batch=1000000, noise_mode='const'):
    """Density grid for marching cubes (gen_samples_next3d.py:208-238) -> float32 numpy [R,R,R], flipped and trimmed like the
    script's.  The tri-planes are computed ONCE (the script's G.sample re-runs the three backbones for every 1M-point chunk: 17
    times at 256^3, 135 times at 512^3), the query points are generated inside the decoding kernel and only sigma is decoded.
    max_batch is kept for API compatibility with the script's chunk size."""
    return _sigma_grid(G, ws, v, shape_res, noise_mode).cpu().numpy()


def extract_mesh(G, ws, v, shape_res=512, level=10.0, noise_mode='const'):
    """Mesh of the density grid of extract_sigma_grid at `level` (the reference's shape_utils.py default 10) -> (verts float32
    [V, 3], faces int32 [F, 3]) CUDA tensors (next3d_b200.isosurface.marching_cubes); the grid never leaves the device.  The
    -1000 border trim keeps the mesh closed."""
    from .isosurface import marching_cubes
    return marching_cubes(_sigma_grid(G, ws, v, shape_res, noise_mode), level)


# ------------------------------------------------------------------------------------------------ sample sheets (gen_samples_next3d.py)
SHEET_YAWS = (0.4, 0.0, -0.4)          # gen_samples_next3d.py:187-188: three yaws, left to right on the sheet, all at pitch -0.2
SHEET_PITCH = -0.2
NUM_WS = 28                            # mapping_ws of the backbone (triplane_next3d.py:65)


def _view_cameras(G, angles, fov_deg):
    """camera_params float32 [len(angles), 25] of the views angles = [(horizontal, vertical)]: look_at_pose(horizontal, vertical)
    looking at rendering_kwargs['avg_camera_pivot'] (default [0, 0, 0]) from radius rendering_kwargs['avg_camera_radius'] (default
    2.7), with FOV_to_intrinsics(fov_deg)."""
    rk = G.rendering_kwargs
    pivot = torch.tensor(rk.get('avg_camera_pivot', [0, 0, 0]))
    radius = rk.get('avg_camera_radius', 2.7)
    out = torch.empty(len(angles), 25)
    out[:, 16:] = camera.fov_to_intrinsics(fov_deg).reshape(9)
    for n, (horizontal, vertical) in enumerate(angles):
        out[n, :16] = camera.look_at_pose(horizontal, vertical, pivot, radius).reshape(16)
    return out


def sample_sheet_cameras(G, fov_deg=18.837):
    """(cams [3, 25], cond [1, 25]) float32: the camera_params of yaws +0.4, 0, -0.4 at pitch -0.2 and the frontal conditioning_params
    of gen_samples_next3d.py:186-196 (np.pi / 2 + angle, where the video script writes 3.14 / 2), with _view_cameras' pivot, radius
    and FOV_to_intrinsics(fov_deg).  fov_deg may be an int or a float: the script declares --fov-deg as an int with the default
    18.837, which click casts to 18 when the option is omitted."""
    cams = _view_cameras(G, [(np.pi / 2 + yaw, np.pi / 2 + SHEET_PITCH) for yaw in SHEET_YAWS], fov_deg)
    return cams, _view_cameras(G, [(np.pi / 2, np.pi / 2)], fov_deg)


def seed_latents(seeds, z_dim):
    """z [S, z_dim] float64: row s is np.random.RandomState(seeds[s]).randn(1, z_dim), the latent every inference script draws per seed."""
    return torch.from_numpy(np.stack([np.random.RandomState(seed).randn(1, z_dim)[0] for seed in seeds]))


def sample_sheet_ws(G, seeds, truncation_psi=1, truncation_cutoff=14, fov_deg=18.837):
    """ws [S, 28, 512] on the generator's device: row s is the script's G.mapping(RandomState(seeds[s]).randn(1, z_dim), cond,
    truncation_psi, truncation_cutoff) (gen_samples_next3d.py:184, 198) with cond from sample_sheet_cameras.  One mapping call maps all
    seeds: on CUDA, n3d_mapping computes each row in its own thread block, so a row does not depend on the others."""
    if len(seeds) == 0:
        raise ValueError('seeds: no seed given')
    device = next(G.parameters()).device
    _, cond = sample_sheet_cameras(G, fov_deg)
    z = seed_latents(seeds, G.z_dim).to(device)
    return G.mapping(z, cond.to(device).expand(len(seeds), -1), truncation_psi=truncation_psi, truncation_cutoff=truncation_cutoff)


def sheet_u8(front, views):
    """uint8 sample sheets [B, H, 3 W, 3] of B heads from their images at yaw +0.4, front [B, 3, H, W], and at yaws 0 and -0.4, views
    [2 B, 3, H, W] (view n of head n // 2): the script's torch.cat(imgs, dim=2) of its uint8 images (gen_samples_next3d.py:201-204),
    on whatever device the images are."""
    B, _, H, W = front.shape
    side = to_uint8_hwc(views).reshape(B, 2, H, W, 3).transpose(1, 2).reshape(B, H, 2 * W, 3)
    return torch.cat([to_uint8_hwc(front), side], 2)


def _check_heads(G, ws, v, batch, shape_res):
    """Refuse bad arguments of the sample-sheet and coloured-mesh drivers (ValueError naming the argument)."""
    if ws.ndim != 3 or tuple(ws.shape[1:]) != (NUM_WS, G.w_dim):
        raise ValueError(f'ws must be [S, {NUM_WS}, {G.w_dim}], got {tuple(ws.shape)}')
    if ws.shape[0] == 0:
        raise ValueError('ws holds no seed (S = 0)')
    if batch < 1:
        raise ValueError(f'batch must be at least 1, got {batch}')
    if shape_res < 2:
        raise ValueError(f'shape_res must be at least 2, got {shape_res}')
    if v.ndim != 3 or v.shape[0] != 1:
        raise ValueError(f'v must be one mesh [1, V, 3] (the script renders every seed with the same mesh), got {tuple(v.shape)}')


def render_sample_sheets(G, ws, v, fov_deg=18.837, batch=9, shapes=False, shape_res=512, seed=None, sampler_noise=None, plan=None):
    """gen_samples_next3d.py:182-238 for the seeds of ws [S, 28, 512] (sample_sheet_ws) and one mesh v [1, V, 3]: yields
    (i, sheet, sigmas) in seed order, for the seeds the plan owns (a head_plan of S heads; default: all of them in calls of
    B = max(1, batch // 3) heads).  sheet: uint8 [H, 3 W, 3] numpy, the script's three yaws side by side (sheet_u8);
    sigmas: float32 [R, R, R] numpy with R = shape_res, equal to extract_sigma_grid(G, ws[i:i + 1], v, shape_res), or None unless
    `shapes`.  Each call renders its heads' three yaws with _head_views_step -- one synthesis call with cache_backbone for yaw +0.4,
    one render_views call for the other two -- and each head's density grid is decoded from its cached planes, so the backbones run
    once per head (the script runs them three times for the sheet and once per 1M-point chunk for the shape).  The last call is
    padded by repeating its last head.  The device->host copy of call k overlaps call k+1.  With G.use_cuda_graph (and no
    sampler_noise) the calls replay CUDA graphs.  The driver replaces whatever heads the generator had cached.
    `seed`: call c of the single-process run draws sampler seeds seed + 2 c (synthesis) and seed + 2 c + 1 (render_views); None =
    fresh random seeds.  `sampler_noise=(u_coarse [3 S, M, Dc, 1], u_fine [3 S, M, Df])` rows are indexed by the global image id
    3 i + yaw (yaw 0, 1, 2 = +0.4, 0, -0.4), in place of `seed`.  ValueError, before any device work, for an empty or misshapen ws,
    batch < 1, shape_res < 2 or a v batch other than 1."""
    _check_heads(G, ws, v, batch, shape_res)
    device = next(G.parameters()).device
    plan = head_plan(ws.shape[0], max(1, batch // 3)) if plan is None else plan
    sheets = _sheets_step(G, plan, ws, v, fov_deg, shapes, shape_res, device, seed, sampler_noise)

    def step(k, idx):
        u8, _, sigmas = sheets(k, idx)
        return (u8, sigmas) if shapes else u8
    batches = ((step(k, plan.frames(k)), plan.keep(k)[1]) for k in range(plan.steps))     # whole calls: keep(k) is (0, n)
    return ((plan.own[0] + i, *(item if shapes else (item, None))) for i, item in enumerate(_to_host(batches, device)))


def render_sample_sheets_sharded(G, ws, v, fov_deg=18.837, batch=9, shapes=False, shape_res=512, seed=0, sampler_noise=None, out=None,
                                 device=None):
    """render_sample_sheets over the GPUs of a box (one process per GPU, as render_frames_sharded): the seeds are split with
    shard_plan (plan.batch heads per step, batch // 3 as the bound) and the sheets gathered to rank 0.  -> (sheets, sigmas):
    sheets is the [S, H, 3 W, 3] uint8 host tensor on rank 0 (`out` if given), None elsewhere, filled in stream order as in
    render_frames_sharded; sigmas is {i: float32 [R, R, R] numpy} for this rank's own seeds i (empty unless `shapes`; the grids are not
    gathered: one 512^3 grid is 512 MB), complete on return.  Step k of rank r draws sampler seeds seed + 2 (r * steps + k) and one
    more; `sampler_noise` rows are indexed 3 i + yaw by the global seed index i, so the results do not depend on the number of ranks.
    Refusals as in render_sample_sheets."""
    _check_heads(G, ws, v, batch, shape_res)
    device = device or next(G.parameters()).device
    cuda = torch.device(device).type == 'cuda'
    plan = shard_plan(ws.shape[0], max(1, batch // 3))
    sheets = _sheets_step(G, plan, ws, v, fov_deg, shapes, shape_res, device, seed, sampler_noise)
    grids = {}

    def step(k, idx):
        u8, new, sigmas = sheets(k, idx)
        for b, i in enumerate(new):
            grids[i] = torch.empty(sigmas[b].shape, pin_memory=cuda)
            grids[i].copy_(sigmas[b], non_blocking=cuda)
        return u8
    res = G.img_resolution
    host = _gather_frames(plan, step, res, 3 * res, device, out)
    if cuda and grids:
        torch.cuda.current_stream(device).synchronize()
    return host, {i: g.numpy() for i, g in grids.items()}


def _head_views_step(G, plan, ws, cams, meshes, device, seed, sampler_noise, mesh_ids=None):
    """step(k, idx) -> the float images [len(idx), V, 3, H, W] of the heads ws[idx] in V views: one synthesis call with
    cache_backbone renders view 0 and keeps the heads, and for V > 1 one render_views call renders views 1 .. V - 1 from the cached
    planes (view n of head idx[n // (V - 1)]).  cams: [V, 25] shared by every head, or [N, V, 25] per head; meshes: one mesh
    [1, Nv, 3] for every head, or [M, Nv, 3] with mesh_ids[i] the mesh of head i.  The two calls of step k draw the sampler seed
    ids 2 c and 2 c + 1 of its call c = plan.step_id(k); the rows of the per-image uniforms are V i + view for head i."""
    cams = cams.to(device, torch.float32)
    meshes = meshes.to(device, torch.float32)
    per_head, V = cams.ndim == 3, cams.shape[-2]

    def step(k, idx):
        B, s = len(idx), 2 * plan.step_id(k)
        w = ws[idx].to(device, torch.float32, non_blocking=True)
        v = meshes.expand(B, -1, -1) if mesh_ids is None else meshes[mesh_ids[idx].to(device)]
        front = G.synthesis(w, cams[idx, 0] if per_head else cams[:1].expand(B, -1), v, noise_mode='const', cache_backbone=True,
                            **_sampler_kw(seed, sampler_noise, s, [V * i for i in idx]))['image'][:, None]
        if V == 1:
            return front
        more = G.render_views(cams[idx, 1:].reshape(-1, 25) if per_head else cams[1:].repeat(B, 1),
                              **_sampler_kw(seed, sampler_noise, s + 1, [V * i + j for i in idx for j in range(1, V)]))['image']
        return torch.cat([front, more.reshape(B, V - 1, *more.shape[1:])], 1)
    return step


def _sheets_step(G, plan, ws, v, fov_deg, shapes, shape_res, device, seed, sampler_noise):
    """step(k, idx) -> (uint8 sheets [len(idx), H, 3 W, 3], new, float32 density grids [len(new), R, R, R] or None) of the heads
    ws[idx]: their three yaws from _head_views_step, and with `shapes` the grid of each head in `new` -- this rank's heads of the
    step that have none yet -- decoded from its cached planes."""
    views = _head_views_step(G, plan, ws, sample_sheet_cameras(G, fov_deg)[0], v, device, seed, sampler_noise)
    lo, hi = plan.spans[plan.rank]
    done = set()

    def step(k, idx):
        images = views(k, idx)
        # a prefix of idx: a short tail repeats the last head, a rank past its span repeats a head it has done, a rank without heads
        # repeats the previous rank's last
        new = [i for i in dict.fromkeys(idx) if lo <= i < hi and i not in done] if shapes else []
        done.update(new)
        sigmas = torch.empty(len(new), shape_res, shape_res, shape_res, device=device) if new else None
        for b in range(len(new)):
            G._get_engine().cached_sigma_grid(b, shape_res, sigmas[b])
        return sheet_u8(images[:, 0], images[:, 1:].flatten(0, 1)), new, sigmas
    return step


# ------------------------------------------------------------------------------------------------------------- multi-view datasets
def dataset_heads(seeds, expressions=1, num_meshes=1):
    """(head seeds, head expressions): one head per (seed, expression), seed-major.  With one mesh every seed has expression 0;
    with num_meshes driving frames, seed s takes `expressions` distinct frame indices, sorted, drawn by
    np.random.RandomState([s, 0]).choice(num_meshes, expressions, replace=False)."""
    if expressions < 1 or expressions > num_meshes:
        raise ValueError(f'expressions must be in 1..{num_meshes} (the driving frames), got {expressions}')
    hs, he = [], []
    for s in seeds:
        ex = [0] if num_meshes == 1 else sorted(int(e) for e in np.random.RandomState([s, 0]).choice(num_meshes, expressions, replace=False))
        hs += [int(s)] * len(ex)
        he += ex
    return hs, he


def dataset_cameras(G, seeds, views, yaw_std=0.3, pitch_std=0.155, fov_deg=18.837):
    """camera_params float32 [S, views, 25] of each seed's views: view 0 looks from the front (sample_sheet_cameras' conditioning
    camera); view v >= 1 is GaussianCameraPoseSampler's draw -- yaw pi/2 + yaw_std * n1 and pitch pi/2 + pitch_std * n2, the
    pitch clamped to (1e-5, pi - 1e-5) -- with (n1, n2) = np.random.RandomState([seed, v]).randn(2), looking at the pivot from
    avg_camera_radius, with FOV_to_intrinsics(fov_deg) (_view_cameras)."""
    angles = []
    for s in seeds:
        for v in range(views):
            n1, n2 = np.random.RandomState([int(s), v]).randn(2) if v else (0.0, 0.0)
            angles.append((np.pi / 2 + yaw_std * n1, float(np.clip(np.pi / 2 + pitch_std * n2, 1e-5, np.pi - 1e-5))))
    return _view_cameras(G, angles, fov_deg).reshape(len(seeds), views, 25)


def dataset_image_name(i):
    """dataset_tool.py's name of image i: '00000/img00000000.png', a folder per 1000 images."""
    return f'{i // 1000:05d}/img{i:08d}.png'


def render_dataset(G, ws, meshes, mesh_ids, cams, plan, seed=None):
    """Multi-view images of the heads of a head_plan: ws [N, 28, 512] and cams [N, V, 25] per head, meshes [M, Nv, 3] and
    mesh_ids[h], the mesh of head h.  Each call renders its heads' V views with _head_views_step: one synthesis call with
    cache_backbone for view 0, one render_views call for the other V - 1 views, with sampler seeds seed + 2 c and seed + 2 c + 1
    for the single-process call index c.  Yields (first head, uint8 frames [n V, H, W, 3] on the generator's device) for the n
    heads of each call that the plan owns, head-major and view-minor; a short last call repeats its last head, as render_sample_sheets
    does."""
    device = next(G.parameters()).device
    step = _head_views_step(G, plan, ws, cams, meshes, device, seed, None, torch.as_tensor(mesh_ids, dtype=torch.long))
    for k in range(plan.steps):
        idx, (lo, hi) = plan.frames(k), plan.keep(k)
        yield idx[lo], to_uint8_hwc(step(k, idx)[lo:hi].flatten(0, 1))


# ------------------------------------------------------------------------------------------------------------- coloured meshes
# The views baked onto a mesh: yaws -0.8 .. 0.8 at the sample sheets' pitch -0.2, and three yaws at pitch +0.2 that see under the
# chin and brows.  Beyond |yaw| 0.8 (2.7 sigma of gen_dataset's default yaw spread 0.3) the generator leaves its training poses
# and the images stop being trustworthy (DESIGN.md section 3.8).
BAKE_VIEWS = tuple((yaw, SHEET_PITCH) for yaw in (-0.8, -0.4, 0.0, 0.4, 0.8)) + tuple((yaw, 0.2) for yaw in (-0.4, 0.0, 0.4))
BAKE_BATCH = 3                         # heads per rendering call of coloured_meshes


def bake_cameras(G, fov_deg=18.837):
    """camera_params float32 [len(BAKE_VIEWS), 25] of the bake views: look_at_pose(pi / 2 + yaw, pi / 2 + pitch) around
    avg_camera_pivot from avg_camera_radius with FOV_to_intrinsics(fov_deg) (_view_cameras, as the sheets' views)."""
    return _view_cameras(G, [(np.pi / 2 + yaw, np.pi / 2 + pitch) for yaw, pitch in BAKE_VIEWS], fov_deg)


def coloured_meshes(G, ws, v, plan=None, batch=BAKE_BATCH, shape_res=512, level=10.0, fov_deg=18.837, seed=0):
    """Coloured meshes of the heads ws [S, 28, 512] (sample_sheet_ws) with one mesh v [1, V, 3]: yields (i, verts float32 [V, 3],
    faces int32 [F, 3], colors uint8 [V, 3]) CUDA tensors in head order, for the heads the plan owns (a head_plan of heads in calls
    of `batch`; default: all of them).  Each call renders the bake views of its heads with _head_views_step (one caching synthesis
    call for bake view 0, one render_views call for the others; sampler seeds seed + 2 c and seed + 2 c + 1 for the single-process
    call index c); each head's density grid comes from its cached planes, is meshed by marching cubes (extract_mesh's mesh), and
    the views are baked onto the vertices (next3d_b200.bake), with the decoder's colour at the vertex where no view sees it.  A
    short last call repeats its last head.  Refusals as in render_sample_sheets."""
    from .bake import bake_vertex_colors, mesh_zbuffer, world_points
    from .isosurface import marching_cubes
    _check_heads(G, ws, v, batch, shape_res)
    device = next(G.parameters()).device
    plan = head_plan(ws.shape[0], batch) if plan is None else plan
    eng = G._get_engine()
    cams = bake_cameras(G, fov_deg).to(device)
    views = _head_views_step(G, plan, ws, cams, v, device, seed, None)
    grid = torch.empty(shape_res, shape_res, shape_res, device=device) if plan.steps else None
    box = G.rendering_kwargs['box_warp']
    for k in range(plan.steps):
        idx, (lo, hi) = plan.frames(k), plan.keep(k)
        images = views(k, idx)                                                       # [B, views, 3, H, W]
        for b in range(lo, hi):
            eng.cached_sigma_grid(b, shape_res, grid)
            verts, faces = marching_cubes(grid, level)
            world = world_points(verts, shape_res, box)
            _, feat = eng.cached_sample_points(b, world)
            zbuf = mesh_zbuffer(world, faces, cams, images.shape[-2], images.shape[-1])
            yield idx[b], verts, faces, bake_vertex_colors(verts, world, grid, cams, images[b], zbuf, feat, box)


def extract_coloured_mesh(G, ws, v, shape_res=512, level=10.0, fov_deg=18.837, seed=0):
    """The coloured mesh of one head ws [1, 28, 512] with mesh v [1, V, 3] -> (verts float32 [V, 3], faces int32 [F, 3], colors
    uint8 [V, 3]) CUDA tensors: the geometry of extract_mesh(G, ws, v, shape_res, level), the colours of coloured_meshes (its
    first call, sampler seeds seed and seed + 1)."""
    _, verts, faces, colors = next(coloured_meshes(G, ws[:1], v, batch=1, shape_res=shape_res, level=level, fov_deg=fov_deg, seed=seed))
    return verts, faces, colors
