"""Standalone inference scripts: `python -m next3d_b200 {gen_samples,gen_videos,reenact} ...`, `gen_dataset` (multi-view
training images in dataset_tool.py's layout), `shape_utils` (the reference's .mrc -> .ply converter, marching cubes on the GPU) and
`gen_meshes` (one coloured .ply mesh per seed: gen_samples' shape, meshed on the GPU, with the rendered views baked onto its
vertices).

The three subcommands are the reference's gen_samples_next3d.py, gen_videos_next3d.py and reenact_avatar_next3d.py with their option
names, defaults and output file names, run on a network pickle read by next3d_b200.legacy (no reference checkout, no pickled code
run) and rendered by the batched drivers of next3d_b200.drivers on one CUDA device.  Differences from the scripts:
  * `--network` is a local file (no URL download);
  * the ray sampler draws its uniforms from seed 0 (the scripts use fresh torch.rand draws), so a run is reproducible;
  * `--lms_cond True` is required: the generator reads the 68 landmarks that follow the mesh vertices (load_lms), and without them
    the scripts fail as well;
  * `--shape-format .ply` (mesh the .mrc grids with `shape_utils` instead) and `--cfg` other than FFHQ are refused, and so is `--interpolate False` with a
    grid larger than 1x1 (every cell would show the same head);
  * mp4 files are written with imageio (libx264 at the scripts' bitrates); without it the video commands refuse before loading
    the network.  `--encoder n3d` writes them with this package's H.264 encoder on the GPU instead (next3d_b200.video: constant
    `--qp`, default 18, integer-pel motion, no deblocking; INTEGRATION.md section 0) and never imports imageio.  With
    `--bitrate` (`script`: the scripts' 10M / 12M, or a rate such as 8M) it writes the rate-controlled stream instead: QP chosen
    on the GPU per frame, quarter-sample motion and deblocking.

Under torchrun (`torchrun --nproc-per-node N -m next3d_b200 ...`) every rank loads the network and renders its share on its own
GPU (LOCAL_RANK), with a gloo process group for the little that crosses ranks.  A video is split into whole GOPs (`--gop`,
default 60): each rank renders exactly the calls the single-process run makes for its frames (same images, padding and sampler
seed), encodes them with `--encoder n3d` on its GPU, and rank 0 gathers the coded samples and writes the one MP4, so the files are
byte for byte those of one process (with `--bitrate`, each rank's share starts its own rate controller instead: a valid file, not
the same bytes).  gen_samples splits the seeds in whole calls and every rank writes its own seeds' files.  `--encoder imageio` is
refused under torchrun.
"""
import argparse
import contextlib
import datetime
import glob
import io
import math
import os
import re
import sys

import torch

SAMPLER_SEED = 0
DIST_TIMEOUT = datetime.timedelta(minutes=60)        # the longest a rank waits for the others at a collective


def _bool(s):
    v = s.strip().lower()
    if v in ('1', 'true', 't', 'yes', 'y', 'on'):
        return True
    if v in ('0', 'false', 'f', 'no', 'n', 'off'):
        return False
    raise argparse.ArgumentTypeError(f'{s!r} is not a valid boolean')


def _range(s):
    """'0,1,4-6' -> [0, 1, 4, 5, 6] (parse_range of the scripts)."""
    out = []
    for p in s.split(','):
        m = re.match(r'^(\d+)-(\d+)$', p)
        out.extend(range(int(m.group(1)), int(m.group(2)) + 1) if m else [int(p)])
    return out


def _tuple(s):
    """'4x2' or '4,2' -> (4, 2) (parse_tuple of the scripts)."""
    m = re.match(r'^(\d+)[x,](\d+)$', s)
    if not m:
        raise argparse.ArgumentTypeError(f'cannot parse tuple {s}')
    return int(m.group(1)), int(m.group(2))


def _parser():
    p = argparse.ArgumentParser(prog='python -m next3d_b200', description=__doc__.split('\n')[0])
    sub = p.add_subparsers(dest='command', required=True)
    # --fov-deg is declared type=int with the default 18.837 in the scripts, which click casts to 18 when the option is omitted
    s = sub.add_parser('gen_samples', help='sample sheets (three yaws per seed) and optional .mrc density grids')
    s.add_argument('--network', required=True, help='network pickle (local file)')
    s.add_argument('--seeds', type=_range, required=True)
    s.add_argument('--obj_path', required=True)
    s.add_argument('--lms_path', required=True)
    s.add_argument('--trunc', dest='truncation_psi', type=float, default=1)
    s.add_argument('--trunc-cutoff', dest='truncation_cutoff', type=int, default=14)
    s.add_argument('--outdir', required=True)
    s.add_argument('--shapes', type=_bool, default=False)
    s.add_argument('--shape-res', dest='shape_res', type=int, default=512)
    s.add_argument('--fov-deg', dest='fov_deg', type=int, default=18)
    s.add_argument('--shape-format', dest='shape_format', choices=['.mrc', '.ply'], default='.mrc')
    s.add_argument('--lms_cond', type=_bool, default=False)
    s.add_argument('--reload_modules', type=_bool, default=False)

    v = sub.add_parser('gen_videos', help='latent interpolation (or one-head orbit) videos')
    v.add_argument('--network', required=True, help='network pickle (local file)')
    v.add_argument('--seeds', type=_range, required=True)
    v.add_argument('--obj_path', required=True)
    v.add_argument('--lms_path', required=True)
    v.add_argument('--shuffle-seed', dest='shuffle_seed', type=int, default=None)
    v.add_argument('--grid', type=_tuple, default=(1, 1))
    v.add_argument('--num-keyframes', dest='num_keyframes', type=int, default=None)
    v.add_argument('--w-frames', dest='w_frames', type=int, default=240)
    v.add_argument('--trunc', dest='truncation_psi', type=float, default=1)
    v.add_argument('--trunc-cutoff', dest='truncation_cutoff', type=int, default=14)
    v.add_argument('--outdir', required=True)
    v.add_argument('--reload_modules', type=_bool, default=False)
    v.add_argument('--cfg', choices=['FFHQ', 'AFHQ', 'Shapenet'], default='FFHQ')
    v.add_argument('--image_mode', choices=['image', 'image_depth', 'image_raw'], default='image')
    v.add_argument('--sample_mult', dest='sampling_multiplier', type=float, default=2)
    v.add_argument('--nrr', type=int, default=None)
    v.add_argument('--interpolate', type=_bool, default=True)
    v.add_argument('--save_root', default=None)
    v.add_argument('--lms_cond', type=_bool, default=False)
    _encoder_args(v)

    r = sub.add_parser('reenact', help='drive one or more identities with a tracked mesh sequence')
    r.add_argument('--drive_root', required=True)
    r.add_argument('--fname', default='reenact.mp4')
    r.add_argument('--network', required=True, help='network pickle (local file)')
    r.add_argument('--grid', dest='grid_dims', type=_tuple, default=(1, 1))
    r.add_argument('--seeds', type=_range, required=True)
    r.add_argument('--outdir', required=True)
    r.add_argument('--fov-deg', dest='fov_deg', type=int, default=18)
    r.add_argument('--trunc', dest='truncation_psi', type=float, default=1)
    r.add_argument('--trunc-cutoff', dest='truncation_cutoff', type=int, default=14)
    r.add_argument('--reload_modules', type=_bool, default=False)
    r.add_argument('--lms_cond', type=_bool, default=False)
    r.add_argument('--fixed_camera', type=_bool, default=False)
    r.add_argument('--num_frames', type=int, default=500)
    _encoder_args(r)

    d = sub.add_parser('gen_dataset', help="multi-view images with camera labels, meshes and landmarks, in dataset_tool.py's layout")
    d.add_argument('--network', required=True, help='network pickle (local file)')
    d.add_argument('--seeds', type=_range, required=True)
    d.add_argument('--views', type=int, default=8, help='images per head; view 0 is frontal, the others Gaussian around the pivot')
    d.add_argument('--obj_path', default=None)
    d.add_argument('--lms_path', default=None)
    d.add_argument('--drive_root', default=None, help='driving directory (as reenact): expressions are drawn from its frames')
    d.add_argument('--expressions', type=int, default=None, help='heads per seed, each with another driving frame (needs --drive_root)')
    d.add_argument('--yaw-std', dest='yaw_std', type=float, default=0.3)
    d.add_argument('--pitch-std', dest='pitch_std', type=float, default=0.155)
    d.add_argument('--trunc', dest='truncation_psi', type=float, default=1)
    d.add_argument('--trunc-cutoff', dest='truncation_cutoff', type=int, default=14)
    d.add_argument('--fov-deg', dest='fov_deg', type=float, default=18.837)
    d.add_argument('--outdir', required=True)
    d.add_argument('--batch', type=int, default=4, help='heads per rendering call')
    d.add_argument('--reload_modules', type=_bool, default=False)
    d.add_argument('--lms_cond', type=_bool, default=False)

    m = sub.add_parser('shape_utils', help=".mrc density grids -> .ply meshes (the reference's shape_utils.py), marching cubes on the GPU")
    m.add_argument('input_mrc_path', help='an .mrc file, or a directory whose *.mrc files are all converted')
    m.add_argument('--level', type=float, default=10, help='the isosurface level for marching cubes')

    c = sub.add_parser('gen_meshes', help='coloured .ply meshes: the shape of gen_samples meshed on the GPU, the rendered views baked '
                                          'onto its vertices')
    c.add_argument('--network', required=True, help='network pickle (local file)')
    c.add_argument('--seeds', type=_range, required=True)
    c.add_argument('--obj_path', default=None)
    c.add_argument('--lms_path', default=None)
    c.add_argument('--trunc', dest='truncation_psi', type=float, default=1)
    c.add_argument('--trunc-cutoff', dest='truncation_cutoff', type=int, default=14)
    c.add_argument('--fov-deg', dest='fov_deg', type=float, default=18, help="as gen_samples (whose omitted --fov-deg is 18)")
    c.add_argument('--shape-res', dest='shape_res', type=int, default=512)
    c.add_argument('--level', type=float, default=10, help='the isosurface level for marching cubes')
    c.add_argument('--outdir', required=True)
    c.add_argument('--reload_modules', type=_bool, default=False)
    c.add_argument('--lms_cond', type=_bool, default=False)
    return p


def _encoder_args(p):
    p.add_argument('--encoder', choices=['imageio', 'n3d'], default='imageio',
                   help='imageio: libx264 through imageio (the scripts); n3d: the sm_90a H.264 encoder of next3d_b200.video')
    p.add_argument('--qp', type=int, default=None, help='constant quantiser 0..51 of --encoder n3d (lower = larger, closer; default 18)')
    p.add_argument('--bitrate', default=None,
                   help="--encoder n3d at a bitrate instead of a constant QP: 'script' (the scripts' rate per video) or bits/s "
                        "such as 8M or 800k")
    p.add_argument('--gop', type=int, default=None,
                   help='--encoder n3d: an IDR frame every N frames (default 60); under torchrun the ranks split a video in whole GOPs')


def _refuse(msg):
    raise SystemExit(f'next3d_b200: {msg}')


def _imageio():
    try:
        import imageio
    except ImportError:
        _refuse('writing mp4 videos needs the imageio package (with its ffmpeg plugin), which cannot be imported; '
                'or pass --encoder n3d')
    return imageio


def _video_writer(args):
    """write(path, fps, bitrate, frames, shard) of the chosen --encoder, checked before the network is loaded: imageio writes the
    host frames of frames(), n3d the video of shard(gop, rank, world) (a drivers.*_video_shard) through write_video_sharded."""
    if args.gop is not None and args.encoder != 'n3d':
        _refuse('--gop sets the GOP of --encoder n3d')
    if args.gop is not None and args.gop < 1:
        _refuse(f'--gop {args.gop}: a GOP holds at least one frame')
    if args.encoder == 'imageio' and _world() > 1:
        _refuse('--encoder imageio writes on one process: under torchrun pass --encoder n3d')
    gop = 60 if args.gop is None else args.gop
    if args.bitrate is not None:
        if args.encoder != 'n3d':
            _refuse('--bitrate selects the rate-controlled stream of --encoder n3d; imageio already writes at the scripts\' rates')
        if args.qp is not None:
            _refuse('--bitrate and --qp exclude each other: the rate controller chooses the QP')
        rate = None
        if args.bitrate != 'script':
            from .video import parse_bitrate
            try:
                rate = parse_bitrate(args.bitrate)
            except ValueError as e:
                _refuse(f'--bitrate: {e}')
        return lambda path, fps, bitrate, frames, shard: _write_video_n3d(path, shard, fps, gop, None, rate or bitrate)
    if args.encoder == 'imageio':
        imageio = _imageio()
        return lambda path, fps, bitrate, frames, shard: _write_video(imageio, path, frames(), fps, bitrate)
    qp = 18 if args.qp is None else args.qp
    if not 0 <= qp <= 51:
        _refuse(f'--qp {qp}: the quantiser is 0..51')
    return lambda path, fps, bitrate, frames, shard: _write_video_n3d(path, shard, fps, gop, qp)


def _world():
    return int(os.environ.get('WORLD_SIZE', '1'))


def _rank():
    from . import distributed as D
    return D.rank_world()


def _load(args):
    from . import legacy
    from .triplane_next3d import TriPlaneGenerator
    print(f'Loading networks from "{args.network}"...')
    with open(args.network, 'rb') as f:
        G = legacy.load_network_pkl(f)['G_ema']
    if args.reload_modules:                                  # the scripts' rebuilt generator reads the eye mask from its PNG again
        G.uv_face_mask = TriPlaneGenerator._load_uv_face_mask()
    return G.to('cuda')


def _mesh(args):
    from . import inputs
    return inputs.load_frame(args.obj_path, args.lms_path).to('cuda')


def _write_video(imageio, path, frames, fps, bitrate):
    writer = imageio.get_writer(path, mode='I', fps=fps, codec='libx264', bitrate=bitrate)
    try:
        for frame in frames:
            writer.append_data(frame)
    finally:
        writer.close()


def _write_video_n3d(path, shard, fps, gop, qp, bitrate=None):
    from . import drivers
    from .video import H264Encoder
    rank, world = _rank()
    kw = dict(qp=qp) if bitrate is None else dict(bitrate=bitrate)
    drivers.write_video_sharded(path, lambda: shard(gop, rank, world),
                                lambda width, height, first: H264Encoder(width, height, fps, gop=gop, first_frame=first, **kw))


def gen_samples(args):
    """gen_samples_next3d.py: seedNNNN.png sheets and, with --shapes, seedNNNN.mrc density grids.  Under torchrun every rank renders
    and writes the seeds of its whole calls (drivers.head_plan)."""
    import PIL.Image
    from . import distributed as D, drivers, mrc
    if args.shape_format == '.ply':
        _refuse('--shape-format .ply: gen_samples writes the script\'s .mrc grids; mesh them with python -m next3d_b200 shape_utils '
                'OUTDIR (marching cubes on the GPU)')
    G = _load(args)
    v = _mesh(args)
    rank, world = _rank()

    def body():
        os.makedirs(args.outdir, exist_ok=True)
        ws = drivers.sample_sheet_ws(G, args.seeds, args.truncation_psi, args.truncation_cutoff, args.fov_deg)
        plan = drivers.head_plan(len(args.seeds), 3, rank, world)
        for i, sheet, sigmas in drivers.render_sample_sheets(G, ws, v, fov_deg=args.fov_deg, shapes=args.shapes, shape_res=args.shape_res,
                                                             seed=SAMPLER_SEED, plan=plan):
            name = os.path.join(args.outdir, f'seed{args.seeds[i]:04d}')
            PIL.Image.fromarray(sheet, 'RGB').save(name + '.png')
            if sigmas is not None:
                mrc.write_mrc(name + '.mrc', sigmas)
    D.run_together(body)


def _check_dataset_args(args):
    if args.views < 1:
        _refuse(f'--views must be at least 1, got {args.views}')
    if args.batch < 1:
        _refuse(f'--batch must be at least 1, got {args.batch}')
    if args.expressions is not None and args.drive_root is None:
        _refuse('--expressions draws driving frames: it needs --drive_root')
    mesh = args.obj_path is not None or args.lms_path is not None
    if mesh and args.drive_root is not None:
        _refuse('give either --obj_path / --lms_path or --drive_root, not both')
    if args.drive_root is None and (args.obj_path is None or args.lms_path is None):
        _refuse('give --obj_path and --lms_path (one expression), or --drive_root')


def _link(src, dst, data=None):
    """dst as a hard link to src, or, without src, a new file of `data`."""
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    if os.path.lexists(dst):
        os.remove(dst)
    if src is None:
        with open(dst, 'wb') as f:
            f.write(data)
    else:
        os.link(src, dst)


def gen_dataset(args):
    """Multi-view images of heads (seed, expression) in dataset_tool.py's layout, which the reference's ImageFolderDataset and
    mesh loader read: images/NNNNN/imgNNNNNNNN.png (head-major, view-minor) with images/dataset.json holding each image's 25
    camera floats, meshes/NNNNN/imgNNNNNNNN.obj and lms/NNNNN/imgNNNNNNNN.txt (each distinct mesh written once per rank and
    hard-linked per image), and heads.npz (seed, expression, ws per head).  PNG files come from the GPU encoder
    (next3d_b200.png).  Under torchrun the heads are split in whole calls and every rank writes its own images; every rank
    computes every label, so rank 0 writes dataset.json and heads.npz."""
    import json
    import numpy as np
    from . import distributed as D, drivers, inputs
    from .png import PngEncoder
    _check_dataset_args(args)
    if args.drive_root is not None:
        sched = drivers.reenact_schedule(args.drive_root, 1 << 30, lms_cond=True)
        sources = list(zip(sched['obj_paths'], sched['lms_paths']))
        if not sources:
            _refuse(f'--drive_root {args.drive_root}: no driving frames')
    else:
        sources = [(args.obj_path, args.lms_path)]
    K = args.expressions or 1
    if K > len(sources):
        _refuse(f'--expressions {K}: the driving directory has {len(sources)} frames')
    G = _load(args)
    rank, world = _rank()

    def body():
        head_seeds, head_exprs = drivers.dataset_heads(args.seeds, K, len(sources))
        used = sorted(set(head_exprs))
        meshes = torch.cat([inputs.load_frame(*sources[e]) for e in used])
        mesh_ids = [used.index(e) for e in head_exprs]
        ws_seed = drivers.sample_sheet_ws(G, args.seeds, args.truncation_psi, args.truncation_cutoff, args.fov_deg)
        row = {s: i for i, s in enumerate(args.seeds)}
        ws = ws_seed[[row[s] for s in head_seeds]]
        cams_seed = drivers.dataset_cameras(G, args.seeds, args.views, args.yaw_std, args.pitch_std, args.fov_deg)
        cams = cams_seed[[row[s] for s in head_seeds]]
        V = args.views
        img_dir, mesh_dir, lms_dir = (os.path.join(args.outdir, d) for d in ('images', 'meshes', 'lms'))
        os.makedirs(img_dir, exist_ok=True)
        if rank == 0:
            labels = [[drivers.dataset_image_name(h * V + v), [float(x) for x in cams[h, v]]] for h in range(len(head_seeds))
                      for v in range(V)]
            with open(os.path.join(img_dir, 'dataset.json'), 'w') as f:
                json.dump({'labels': labels}, f)
            np.savez(os.path.join(args.outdir, 'heads.npz'), seed=np.array(head_seeds, np.int64),
                     expression=np.array(head_exprs, np.int64), ws=ws.float().cpu().numpy())
        plan = drivers.head_plan(len(head_seeds), args.batch, rank, world)
        enc = PngEncoder(G.img_resolution, G.img_resolution, batch=2 * args.batch * V)
        first_link = {}                                  # expression -> this rank's first mesh / landmark files of it
        pending = []                                     # image ids submitted to the encoder, not yet written

        def save(files):
            for data in files:
                i = pending.pop(0)
                name = drivers.dataset_image_name(i)
                with open(os.path.join(img_dir, name), 'wb') as f:
                    f.write(data)
                e = head_exprs[i // V]
                stem = name[:-len('.png')]
                obj, lms = os.path.join(mesh_dir, stem + '.obj'), os.path.join(lms_dir, stem + '.txt')
                if e in first_link:
                    _link(first_link[e][0], obj)
                    _link(first_link[e][1], lms)
                else:
                    _link(None, obj, open(sources[e][0], 'rb').read())
                    _link(None, lms, open(sources[e][1], 'rb').read())
                    first_link[e] = (obj, lms)
        for h0, frames in drivers.render_dataset(G, ws, meshes, mesh_ids, cams, plan, seed=SAMPLER_SEED):
            for i in range(h0 * V, h0 * V + frames.shape[0]):
                os.makedirs(os.path.join(img_dir, drivers.dataset_image_name(i)[:5]), exist_ok=True)
                pending.append(i)
            save(enc.write(frames))
        save(enc.flush())
    D.run_together(body)


def _shape_files(args):
    """The .mrc files shape_utils converts, sorted; the refusals come before any CUDA work."""
    if not math.isfinite(args.level):
        _refuse(f'--level {args.level}: the isosurface level must be finite')
    path = args.input_mrc_path
    if os.path.isdir(path):
        return sorted(glob.glob(os.path.join(path, '*.mrc')))
    if not os.path.exists(path):
        _refuse(f'{path}: no such file or directory')
    if not path.endswith('.mrc'):
        _refuse(f'{path}: shape_utils converts .mrc files (or a directory of them)')
    return [path]


def shape_utils(args):
    """shape_utils.py: each .mrc grid (the file, or every *.mrc directly in the directory) -> stem.ply beside it, meshed at --level
    by next3d_b200.isosurface.  Unlike the script, a single file is meshed at --level too (the script uses level 1 and only
    takes a path ending in .ply).  Under torchrun the ranks split the sorted files (distributed.shard_range)."""
    from . import distributed as D, isosurface, mrc
    files = _shape_files(args)
    if not files:
        print(f'no .mrc files in {args.input_mrc_path}: nothing converted')
        return
    rank, world = _rank()
    a, b = D.shard_range(len(files), rank, world)

    def body():
        for path in files[a:b]:
            out = os.path.splitext(path)[0] + '.ply'
            verts, faces = isosurface.marching_cubes(mrc.read_mrc(path), args.level)
            isosurface.write_ply(out, verts, faces)
            print(f'wrote to {out}')
    D.run_together(body)


def _check_mesh_args(args):
    if not math.isfinite(args.level):
        _refuse(f'--level {args.level}: the isosurface level must be finite')
    if args.shape_res < 2:
        _refuse(f'--shape-res {args.shape_res}: the grid needs at least 2 voxels per side')
    for opt, path in (('--obj_path', args.obj_path), ('--lms_path', args.lms_path)):
        if path is None:
            _refuse(f'{opt} is required: the generator renders every seed with that mesh')
        if not os.path.isfile(path):
            _refuse(f'{opt} {path}: no such file')


def gen_meshes(args):
    """seedNNNN.ply per seed: the density grid of gen_samples --shapes True (same latent and conditioning, sample_sheet_ws) meshed at
    --level by marching cubes, with vertex colours baked from drivers.BAKE_VIEWS (drivers.coloured_meshes).  Under torchrun the
    ranks split the seeds in whole calls (drivers.head_plan), so every file is that of one process."""
    from . import distributed as D, drivers, isosurface
    _check_mesh_args(args)
    G = _load(args)
    v = _mesh(args)
    rank, world = _rank()

    def body():
        os.makedirs(args.outdir, exist_ok=True)
        ws = drivers.sample_sheet_ws(G, args.seeds, args.truncation_psi, args.truncation_cutoff, args.fov_deg)
        plan = drivers.head_plan(len(args.seeds), drivers.BAKE_BATCH, rank, world)
        for i, verts, faces, colors in drivers.coloured_meshes(G, ws, v, plan, shape_res=args.shape_res, level=args.level,
                                                               fov_deg=args.fov_deg, seed=SAMPLER_SEED):
            out = os.path.join(args.outdir, f'seed{args.seeds[i]:04d}.ply')
            isosurface.write_ply(out, verts, faces, colors)
            print(f'wrote to {out}')
    D.run_together(body)


def gen_videos(args):
    """gen_videos_next3d.py: interpolation.mp4 over a --grid of seeds, or with --interpolate False one orbit video SEED.mp4 per seed."""
    from . import drivers
    if args.cfg != 'FFHQ':
        _refuse(f'--cfg {args.cfg}: only the FFHQ generator is implemented')
    if not args.interpolate and tuple(args.grid) != (1, 1):
        _refuse('--interpolate False renders one head per video: use --grid 1x1')
    write = _video_writer(args)
    G = _load(args)
    rk = G.rendering_kwargs
    rk['depth_resolution'] = int(rk['depth_resolution'] * args.sampling_multiplier)
    rk['depth_resolution_importance'] = int(rk['depth_resolution_importance'] * args.sampling_multiplier)
    v = _mesh(args)
    if args.nrr is not None:
        G.neural_rendering_resolution = args.nrr
    psi, cutoff = args.truncation_psi, args.truncation_cutoff
    if cutoff == 0:
        psi = 1.0
    if psi == 1.0:
        cutoff = 14
    os.makedirs(args.outdir, exist_ok=True)
    if args.save_root is not None:
        os.makedirs(args.save_root, exist_ok=True)
    if args.interpolate:
        ws = drivers.grid_keyframes(G, args.seeds, args.grid, args.num_keyframes, args.shuffle_seed, psi, cutoff)
        write(os.path.join(args.outdir, 'interpolation.mp4'), 60, '10M',
              lambda: drivers.render_grid_frames(G, ws, v, args.w_frames, image_mode=args.image_mode, seed=SAMPLER_SEED),
              lambda gop, rank, world: drivers.grid_video_shard(G, ws, v, args.w_frames, gop, rank, world, image_mode=args.image_mode,
                                                                seed=SAMPLER_SEED))
        return
    for seed in args.seeds:
        ws = drivers.grid_keyframes(G, [seed], (1, 1), args.num_keyframes, args.shuffle_seed, psi, cutoff)[0, 0]
        cams = drivers.orbit_camera_params(ws.shape[0] * args.w_frames, torch.tensor(rk['avg_camera_pivot']), rk['avg_camera_radius'])
        write(os.path.join(args.outdir, f'{seed}.mp4'), 60, '12M',
              lambda: drivers.render_orbit(G, ws[:1], cams, v, image_mode=args.image_mode, seed=SAMPLER_SEED),
              lambda gop, rank, world: drivers.orbit_video_shard(G, ws[:1], cams, v, gop, rank, world, image_mode=args.image_mode,
                                                                 seed=SAMPLER_SEED))


def reenact(args):
    """reenact_avatar_next3d.py: --fname (reenact.mp4), the driving photo next to one avatar per seed in a --grid."""
    from . import drivers
    write = _video_writer(args)
    G = _load(args)
    G.rendering_kwargs['return_normal'] = False
    os.makedirs(args.outdir, exist_ok=True)
    _, cond = drivers.sample_sheet_cameras(G, args.fov_deg)
    ws = drivers.sample_sheet_ws(G, args.seeds, args.truncation_psi, args.truncation_cutoff, args.fov_deg)
    fixed = cond if args.fixed_camera else None
    write(os.path.join(args.outdir, args.fname), 30, '12M',
          lambda: drivers.reenact_grid_frames(G, ws, args.drive_root, args.num_frames, args.grid_dims, lms_cond=True,
                                              fixed_camera=fixed, seed=SAMPLER_SEED),
          lambda gop, rank, world: drivers.reenact_grid_video_shard(G, ws, args.drive_root, args.num_frames, args.grid_dims, gop, rank,
                                                                    world, lms_cond=True, fixed_camera=fixed, seed=SAMPLER_SEED))


def main(argv=None):
    args = _parser().parse_args(argv)
    if args.command != 'shape_utils' and not args.lms_cond:
        _refuse('pass --lms_cond True: the generator reads the 68 landmarks that follow the mesh vertices (load_lms)')
    command = {'gen_samples': gen_samples, 'gen_videos': gen_videos, 'reenact': reenact, 'gen_dataset': gen_dataset,
               'shape_utils': shape_utils, 'gen_meshes': gen_meshes}[args.command]
    if args.command == 'gen_dataset':
        _check_dataset_args(args)                            # the refusals, before the process group and the network
    if args.command == 'shape_utils':
        _shape_files(args)                                   # the refusals, before the process group and any CUDA work
    if args.command == 'gen_meshes':
        _check_mesh_args(args)                               # the refusals, before the process group and the network
    if _world() == 1:
        command(args)
        return
    if args.command in ('gen_videos', 'reenact'):
        _video_writer(args)                                  # the refusals, before the process group and the network
    import torch.distributed as dist
    from . import distributed as D
    dist.init_process_group('gloo', rank=int(os.environ['RANK']), world_size=_world(), timeout=DIST_TIMEOUT)
    try:
        torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', '0')))
        quiet = contextlib.nullcontext() if dist.get_rank() == 0 else contextlib.redirect_stdout(io.StringIO())     # rank 0 prints
        try:
            with quiet:
                command(args)
        except D.RankError as e:
            _refuse(str(e))
        dist.barrier()
    finally:
        dist.destroy_process_group()


if __name__ == '__main__':
    main(sys.argv[1:])
