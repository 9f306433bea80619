"""`run_inference` mode of the reference CLI (exps/stage3_root2/test.py:154-225 with `-t run_inference`) on the fused
path: images on disk -> result JSON.

    python -m smap_b200.run_inference -p SMAP.pth [-rp RefineNet.pth] --dataset_path DIR --batch_size 8 --do_flip 1 \
        [--json_name SUFFIX] [--output_dir OUT] [--dataset_name CMU] [--precision {bf16x3,fp16,bf16}] [--jpeg_colour 1]
        [--vis_dir DIR [--vis_format {jpg,png}] [--vis_quality 95] [--vis_3d 1]]

Same flags and the same output file name / schema as the reference ('{OUT}/stage3_root2_run_inference_{data_mode}_{suffix}.json',
test.py:147-152).  Differences, both deliberate: images are visited in sorted path order unless --glob_order 1 (the
reference uses glob order, dataset/custom_dataset.py:16-18).  Decoding, resize, letterbox, normalisation, backbone,
association, lift, RefineNet and the JSON text are produced by libsmap_b200.so: .jpg/.jpeg and .png files the GPU decoders
support are decoded on the GPU (byte-identical to cv2.imread), every other file by cv2.imread as in the reference.  Baseline
JPEGs go through Engine.decode_jpeg; progressive and multi-scan JPEGs through Engine.decode_jpeg_ex, in a batch of their own,
which with --jpeg_colour 1 also takes CMYK, YCCK and RGB JPEGs and every integral sampling (4:1:1, 4:1:0, ...).

Several GPUs: torchrun --nproc_per_node N -m smap_b200.run_inference <same flags>.  With WORLD_SIZE in the environment
(even 1) main() runs run_distributed: torch.distributed over gloo carries only the image list, the NCCL unique id, a
per-step ok flag and the fp16 clamp counts; each rank runs the whole path on device LOCAL_RANK with --batch_size frames
per step (per GPU, as the reference's IMG_PER_GPU), and one NCCL all-gather per step brings the W * B records to rank 0,
which alone writes the file.  The file is byte-identical to the one-GPU file for the same flags and images.

Frames are sharded per step, not in one contiguous block per rank: at step s rank r takes global frames
[(s*W + r)*B, (s*W + r + 1)*B) (step_plan).  The W*B gathered records of a step are then global frames s*W*B ... in
order, so rank 0 appends each step to the result file as it arrives and holds one step of records (W*B * 92,464 B)
whatever the size of the directory.  Contiguous blocks per rank (dist.shard_range) would make rank 0 keep every other
rank's records until its own block ended: gigabytes for a large directory.  In the last step a rank with fewer than B
frames, or none, pads its batch with zero images, so every step runs the same cached graphs and the same fixed-stride
all-gather; the padded slots are never written.

Before each step's exchange is submitted the ranks agree over gloo that every one of them has its frames ready (decoded
and pre-processed), so an unreadable image, a missing checkpoint or an engine error on one rank makes every rank stop
with exit code 1 instead of leaving its peers waiting in the all-gather.
"""
import argparse
import glob
import os
import os.path as osp

import numpy as np
import torch

from .engine import PRECISIONS, RECORD_BYTES, Engine, jpeg_info
from .results import ResultWriter, result_file_name


def list_images(dataset_path, glob_order=False):
    """dataset/custom_dataset.py:16-19 (jpg, png, jpeg; recursive).  Default: sorted, for a reproducible result file;
    glob_order=True keeps the reference's order (per extension, as glob returns them), so that the '3d_pairs' entries
    come in the order the reference writes them and whole files can be compared byte for byte."""
    out = []
    for ext in ("jpg", "png", "jpeg"):
        out.extend(glob.glob(osp.join(dataset_path, "**/*." + ext), recursive=True))
    return out if glob_order else sorted(out)


def image_name(path, dataset_path):
    """dataset/custom_dataset.py:29."""
    return path.rstrip().replace(dataset_path, "").lstrip("/")


def vis_names(paths, dataset_path, ext=".jpg"):
    """-> per image the relative path of its annotated frame under --vis_dir: its image name with the extension replaced
    by ext (".jpg", or ".png" with --vis_format png).  Raises ValueError naming both inputs when two images would write
    the same file (a.png and a.jpg)."""
    names, seen = [], {}
    for p in paths:
        name = osp.splitext(image_name(p, dataset_path))[0] + ext
        if name in seen:
            raise ValueError("--vis_dir: %s and %s would both be written to %s" % (seen[name], p, name))
        seen[name] = p
        names.append(name)
    return names


VIEW3D_MAX_WIDTH = 16384  # the encoder's largest side: a frame of w + h over it has no room for its 3D panel


def write_vis(eng, vis_dir, quality, names, frames, records, scales, view3d=False, fmt="jpg"):
    """Encodes the frames with their skeletons drawn (Engine.encode_jpeg at quality on the device records and scale rows,
    or with fmt "png" Engine.encode_png, lossless) and writes them to vis_dir/names[i], creating subdirectories.
    view3d: each frame with the panel of its 3D skeletons on its right; a frame too wide for that composite raises
    ValueError naming it."""
    kw = {}
    if view3d:
        for name, f in zip(names, frames):
            if f.shape[0] + f.shape[1] > VIEW3D_MAX_WIDTH:
                raise ValueError("--vis_3d: %s is %dx%d, so its composite would be %d pixels wide (at most %d)"
                                 % (name, f.shape[1], f.shape[0], f.shape[0] + f.shape[1], VIEW3D_MAX_WIDTH))
        kw = dict(view3d=True)
    if fmt == "png":
        files = eng.encode_png(frames, records, scales, **kw)
    else:
        files = eng.encode_jpeg(frames, quality, records, scales, **kw)
    for name, data in zip(names, files):
        path = osp.join(vis_dir, name)
        os.makedirs(osp.dirname(path) or ".", exist_ok=True)
        with open(path, "wb") as f:
            f.write(data)


def read_frames(eng, paths, imread, jpeg_colour=False):
    """.jpg/.jpeg files through the GPU JPEG decoder and .png files through the GPU PNG decoder, one batch each; the JPEGs
    decode_jpeg leaves to cv2 that the multi-scan header walk accepts (progressive and multi-scan sequential files, and
    with jpeg_colour CMYK, YCCK, RGB and other samplings) through decode_jpeg_ex, as one more batch, so baseline files
    never wait behind its rounds; the rest, and the files a decoder leaves to cv2, through imread."""
    frames = [None] * len(paths)
    jpegs = {}
    for exts, decode, jpeg in (((".jpg", ".jpeg"), eng.decode_jpeg, True), ((".png",), eng.decode_png, False)):
        sel = [i for i, p in enumerate(paths) if p.lower().endswith(exts)]
        if sel:
            files = []
            for i in sel:
                with open(paths[i], "rb") as f:
                    files.append(f.read())
            for i, b, im in zip(sel, files, decode(files)):
                frames[i] = im
                if jpeg:
                    jpegs[i] = b
    multi = [i for i, b in jpegs.items() if frames[i] is None and jpeg_info(b, scans=True, colour=jpeg_colour)[0] == 0]
    if multi:
        blobs = [jpegs[i] for i in multi]
        for i, im in zip(multi, eng.decode_jpeg_ex(blobs, colour=True) if jpeg_colour else eng.decode_jpeg_ex(blobs)):
            frames[i] = im
    return [imread(p) if im is None else im for p, im in zip(paths, frames)]


def frame_reader(eng, imread=None, jpeg_colour=False):
    """-> read(paths) -> list of uint8 BGR [H,W,3] tensors, the frames run() and run_distributed() pre-process.  imread
    None: read_frames on `eng` with cv2.imread for the files the GPU decoders leave (an unreadable file raises
    RuntimeError("cannot read image ...")); otherwise imread(path) for every file."""
    gpu_decode = imread is None
    if imread is None:
        import cv2

        def imread(p):
            im = cv2.imread(p, cv2.IMREAD_COLOR)
            if im is None:
                raise RuntimeError("cannot read image " + p)
            return im

    colour = dict(jpeg_colour=True) if jpeg_colour else {}

    def read(paths):
        frames = read_frames(eng, paths, imread, **colour) if gpu_decode else [imread(p) for p in paths]
        return [f if torch.is_tensor(f) else torch.from_numpy(np.ascontiguousarray(f)) for f in frames]

    return read


def _load_weights(eng, smap_state_dict, refine_state_dict, precision):
    eng.load_state_dict(smap_state_dict, precision)
    if refine_state_dict is not None:
        eng.load_refine_state_dict(refine_state_dict)
        eng.set_refine(True)


def run(smap_state_dict, dataset_path, output_file, refine_state_dict=None, batch_size=8, do_flip=False, dataset_name="CMU",
        device=0, in_h=512, in_w=832, imread=None, glob_order=False, precision="bf16x3", stats=None, jpeg_colour=False,
        vis_dir=None, vis_quality=95, vis_3d=False, vis_format="jpg"):
    """-> number of images processed.  imread(path) -> uint8 BGR [H,W,3], used for every file; by default .jpg/.jpeg
    and .png files are decoded on the GPU (Engine.decode_jpeg, then Engine.decode_jpeg_ex for the progressive and
    multi-scan JPEGs decode_jpeg leaves, and Engine.decode_png; byte-identical to cv2.imread) and the
    files they do not handle, as every other file, go through cv2.imread(path, IMREAD_COLOR).  jpeg_colour=True: CMYK,
    YCCK and RGB JPEGs and every integral sampling are decoded on the GPU too (Engine.decode_jpeg_ex(colour=True));
    off by default, so those files keep going to cv2.imread.  precision: one of engine.PRECISIONS.  stats (a dict,
    optional) receives "saturation": the fp16 clamp count.  vis_dir: also write every image with its skeletons drawn,
    JPEG-encoded at vis_quality on the GPU (write_vis), to vis_dir/<image name with a .jpg extension>, or with vis_format
    "png" PNG-encoded (lossless) to vis_dir/<image name with a .png extension>; vis_3d: with the panel of its 3D skeletons
    on the right of each frame."""
    if precision not in PRECISIONS:
        raise ValueError("unknown precision %r (choose from %s)" % (precision, ", ".join(PRECISIONS)))
    paths = list_images(dataset_path, glob_order)
    names = vis_names(paths, dataset_path, _vis_ext(vis_format)) if vis_dir else None
    eng = Engine(device, max_batch=batch_size, in_h=in_h, in_w=in_w)
    try:
        _load_weights(eng, smap_state_dict, refine_state_dict, precision)
        read = frame_reader(eng, imread, jpeg_colour)
        host = torch.empty(batch_size, RECORD_BYTES, dtype=torch.uint8).pin_memory()
        with ResultWriter(output_file, dataset_name) as w:
            for lo in range(0, len(paths), batch_size):
                chunk = paths[lo:lo + batch_size]
                frames = read(chunk)
                imgs, scales = eng.preprocess(frames)
                rec = eng.infer_device(imgs, scales.to(imgs.device), do_flip=bool(do_flip))
                host[:len(chunk)].copy_(rec)
                torch.cuda.current_stream().synchronize()
                w.append(host[:len(chunk)], [image_name(p, dataset_path) for p in chunk])
                if vis_dir:
                    write_vis(eng, vis_dir, vis_quality, names[lo:lo + batch_size], frames, rec, scales, vis_3d, vis_format)
        if stats is not None:
            stats["saturation"] = eng.saturation_count()
        return len(paths)
    finally:
        eng.close()


def step_plan(n, world, batch):
    """The schedule of run_distributed for n frames, `world` ranks and `batch` frames per rank and step.  -> one entry per
    step, (shards, slots): shards[r] is the range of global frames rank r takes (empty, or shorter than `batch`, only in
    the last step), slots the gathered slots (r * batch + k) that hold real frames, in global frame order."""
    steps = []
    for lo in range(0, n, world * batch):
        shards = [range(min(n, lo + r * batch), min(n, lo + (r + 1) * batch)) for r in range(world)]
        steps.append((shards, [r * batch + k for r, f in enumerate(shards) for k in range(len(f))]))
    return steps


class RankFailed(RuntimeError):
    """Another rank failed.  pending: this rank's exchange of the step is submitted and can never complete, so its
    engine must not be destroyed (that waits for the device) - the process has to end instead."""

    def __init__(self, failed, pending=False):
        super().__init__("stopped: %d other rank(s) failed" % failed)
        self.pending = pending


def _agree(err, count=0, pending=False):
    """Every rank of the (gloo) default group learns whether any rank has an error; -> the sum of `count` over the ranks.
    Raises err on the rank that has it and RankFailed on the others."""
    import torch.distributed as dist

    t = torch.tensor([0 if err is None else 1, count], dtype=torch.int64)
    dist.all_reduce(t)
    if err is not None:
        raise err
    if t[0]:
        raise RankFailed(int(t[0]), pending)
    return int(t[1])


def drive(n, batch, steps, append):
    """One rank's loop of run_distributed over the steps of step_plan(n, world, batch).  steps: prepare(frames) reads
    this rank's frames of a step (a range of global indices, possibly empty) into a batch of `batch`; submit() starts the
    step's compute and exchange; collect() -> host uint8 [world * batch, RECORD_BYTES], the gathered records once the
    exchange has ended; saturation() -> this rank's fp16 clamp count of its real frames.  append(records, frames) runs
    on rank 0 with the records of the step's real frames and their global indices.  The ranks agree before each
    exchange is submitted, and again before it is waited for, so no rank waits in a collective for a rank that failed;
    an error in collect() or append() is reported at the next agreement.  -> the clamp count summed over the ranks."""
    import torch.distributed as dist

    rank = dist.get_rank()
    err = None
    for shards, slots in step_plan(n, dist.get_world_size(), batch):
        if err is None:
            try:
                steps.prepare(shards[rank])
            except Exception as e:
                err = e
        _agree(err)
        try:
            steps.submit()
        except Exception as e:
            err = e
        _agree(err, pending=True)
        try:
            rec = steps.collect()
            if rank == 0:
                append(rec[slots], [i for f in shards for i in f])
        except Exception as e:
            err = e
    count = 0
    if err is None:
        try:
            count = steps.saturation()
        except Exception as e:
            err = e
    return _agree(err, count)


class _GatherSteps:
    """The GPU side of drive() on one rank: frames read on the rank's engine and pre-processed into fixed buffers (so
    every step replays the same captured graph), padded with zero images to max_batch; the whole path and the all-gather
    with infer_device(gather=True, defer=True); the gathered records copied to a pinned host buffer.  vis(indices, frames,
    records, scales) (optional) runs in collect() with the global indices of the step's real frames, the frames with this rank's slice of the gathered device records."""

    def __init__(self, eng, read, paths, do_flip, vis=None):
        dev = eng.device
        self.eng, self.read, self.paths, self.do_flip, self.B = eng, read, paths, do_flip, eng.max_batch
        self.imgs = torch.empty(self.B, 3, eng.in_h, eng.in_w, device=dev)
        self.scales = torch.empty(self.B, 9, dtype=torch.float64, device=dev)
        self.out = torch.empty(eng.world * self.B, RECORD_BYTES, dtype=torch.uint8, device=dev)
        self.host = torch.empty(eng.world * self.B, RECORD_BYTES, dtype=torch.uint8).pin_memory()
        self.blank = torch.zeros(eng.in_h, eng.in_w, 3, dtype=torch.uint8, device=dev)
        self.n, self.before, self.excess = self.B, None, 0
        self.vis, self.frames, self.indices = vis, [], []

    def prepare(self, frames):
        ims = self.read([self.paths[i] for i in frames]) if len(frames) else []
        _, scales = self.eng.preprocess(ims + [self.blank] * (self.B - len(ims)), out=self.imgs)
        self.scales.copy_(scales)
        self.n = len(ims)
        if self.vis is not None:
            self.frames, self.indices = ims, list(frames)

    def submit(self):
        self.before = self.eng.saturation_count() if self.n < self.B else None
        self.eng.infer_device(self.imgs, self.scales, do_flip=self.do_flip, out=self.out, gather=True, defer=True)

    def collect(self):
        self.eng.gather_sync()
        self.host.copy_(self.out)
        torch.cuda.current_stream().synchronize()
        if self.before is not None:
            padded = self.eng.saturation_count() - self.before
            if padded:  # the zero frames may have been clamped too: count the step's real frames on their own
                if self.n:
                    self.eng.infer_device(self.imgs[:self.n], self.scales[:self.n], do_flip=self.do_flip)
                self.excess += padded
        if self.vis is not None and self.n:
            lo = self.eng.rank * self.B
            self.vis(self.indices, self.frames, self.out[lo:lo + self.n], self.scales[:self.n])
        return self.host

    def saturation(self):
        return self.eng.saturation_count() - self.excess


def run_distributed(smap_state_dict, dataset_path, output_file, refine_state_dict=None, batch_size=8, do_flip=False,
                    dataset_name="CMU", device=None, in_h=512, in_w=832, imread=None, glob_order=False, precision="bf16x3",
                    stats=None, jpeg_colour=False, vis_dir=None, vis_quality=95, vis_3d=False, vis_format="jpg"):
    """run() on every rank of torch.distributed's default group (gloo), with the same arguments; batch_size frames per
    rank and step, device None = LOCAL_RANK.  Rank 0 lists the images and alone writes output_file, byte-identical to
    run()'s; with vis_dir every rank writes the annotated frames of its own shard.  -> number of images;
    stats["saturation"] = the fp16 clamp count summed over the ranks.  When any rank
    fails, every rank raises: the failing one its own error, the others RankFailed."""
    import torch.distributed as dist

    from . import dist as sdist

    if precision not in PRECISIONS:
        raise ValueError("unknown precision %r (choose from %s)" % (precision, ", ".join(PRECISIONS)))
    rank = dist.get_rank()
    device = int(os.environ.get("LOCAL_RANK", 0)) if device is None else device
    eng = writer = err = None
    pending = False
    try:
        try:
            torch.cuda.set_device(device)
            eng = Engine(device, max_batch=batch_size, in_h=in_h, in_w=in_w)
            _load_weights(eng, smap_state_dict, refine_state_dict, precision)
            if rank == 0:
                writer = ResultWriter(output_file, dataset_name)
        except Exception as e:
            err = e
        _agree(err)
        eng.init_comm()
        sdist.sync_tile_table()  # the committed table covers the CLI's input size; this keeps rank 0's choice if not
        box = [list_images(dataset_path, glob_order) if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        paths = box[0]
        vis = None
        if vis_dir:
            names = vis_names(paths, dataset_path, _vis_ext(vis_format))  # the same list on every rank: all refuse a collision

            def vis(indices, frames, records, scales):
                write_vis(eng, vis_dir, vis_quality, [names[i] for i in indices], frames, records, scales, vis_3d, vis_format)
        steps = _GatherSteps(eng, frame_reader(eng, imread, jpeg_colour), paths, bool(do_flip), vis)
        saturation = drive(len(paths), batch_size, steps,
                           lambda rec, frames: writer.append(rec, [image_name(paths[i], dataset_path) for i in frames]))
        if stats is not None:
            stats["saturation"] = saturation
        return len(paths)
    except RankFailed as e:
        pending = e.pending
        raise
    finally:
        if writer is not None:
            writer.close()
        if eng is not None:
            if pending:
                eng._h = None  # its exchange waits for a rank that is gone; the process's exit releases the device
            else:
                eng.close()


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    # the other two modes of the reference (generate_result / generate_train) need its COCO/MuCo dataset loaders, which are
    # out of scope; their device-side piece (register_pred with ground truth) is smapb_lift3d_gt / Engine.lift_gt
    ap.add_argument("--test_mode", "-t", default="run_inference", choices=["run_inference"])
    ap.add_argument("--data_mode", "-d", default="test", choices=["test", "generation"])
    ap.add_argument("--SMAP_path", "-p", default="log/SMAP.pth")
    ap.add_argument("--RefineNet_path", "-rp", default="")
    ap.add_argument("--batch_size", type=int, default=1)
    ap.add_argument("--do_flip", type=float, default=0)
    ap.add_argument("--dataset_path", default="")
    ap.add_argument("--json_name", default="")
    ap.add_argument("--output_dir", default="model_logs/stage3_root2/result")
    ap.add_argument("--dataset_name", default="CMU", help="cfg.DATASET.NAME written as 'model_pattern'")
    ap.add_argument("--glob_order", type=int, default=0, help="1: visit images in the reference's glob order instead of sorted")
    ap.add_argument("--precision", default="bf16x3", choices=list(PRECISIONS),
                    help="convolution precision: bf16x3 (fp32-faithful), fp16 (cost of bf16, 4x finer rounding, range "
                         "+-65504) or bf16 (8-bit mantissa, fp32 range)")
    ap.add_argument("--jpeg_colour", type=int, default=0, choices=[0, 1],
                    help="1: also decode CMYK, YCCK and RGB JPEGs and every integral sampling (4:1:1, 4:1:0, ...) on the "
                         "GPU instead of with cv2.imread")
    ap.add_argument("--vis_dir", default="", help="also write every image with its skeletons drawn, JPEG-encoded on the GPU, "
                                                  "to VIS_DIR/<image name with a .jpg extension>")
    ap.add_argument("--vis_format", default="jpg", choices=["jpg", "png"],
                    help="file format of --vis_dir: jpg (default) or png (lossless, cv2.imencode's bytes), both encoded "
                         "on the GPU; the files are named <image name>.<format>")
    ap.add_argument("--vis_quality", type=int, default=95,
                    help="JPEG quality of --vis_dir, 1..100 (cv2's default 95); JPEG only, --vis_format png ignores it")
    ap.add_argument("--vis_3d", type=int, default=0, choices=[0, 1],
                    help="1: put a panel with the 3D skeletons (pred_3d, seen as lib/visualize/vis.py shows them) on the "
                         "right of every --vis_dir frame")
    a = ap.parse_args(argv)
    if not 1 <= a.vis_quality <= 100:
        ap.error("--vis_quality must be in 1..100")
    if a.vis_3d and not a.vis_dir:
        ap.error("--vis_3d needs --vis_dir")
    if a.vis_format != "jpg" and not a.vis_dir:
        ap.error("--vis_format needs --vis_dir")
    if "WORLD_SIZE" in os.environ:
        return _main_distributed(a)
    try:
        sd, rsd = _load_checkpoints(a)
    except FileNotFoundError as e:
        print(e)
        return 1
    os.makedirs(a.output_dir, exist_ok=True)
    out = result_file_name(a.output_dir, a.test_mode, a.data_mode, a.json_name)
    stats = {}
    n = run(sd, a.dataset_path, out, rsd, a.batch_size, a.do_flip, a.dataset_name, glob_order=bool(a.glob_order),
            precision=a.precision, stats=stats, jpeg_colour=bool(a.jpeg_colour), **_vis_kwargs(a))
    _report(out, n, stats)
    return 0


def _vis_kwargs(a):
    """--vis_dir / --vis_quality / --vis_3d / --vis_format as run()'s keyword arguments; none without --vis_dir, and
    vis_3d and vis_format only when they differ from the default, so that run is called as before without them."""
    kw = dict(vis_dir=a.vis_dir, vis_quality=a.vis_quality) if a.vis_dir else {}
    if a.vis_3d:
        kw["vis_3d"] = True
    if a.vis_format != "jpg":
        kw["vis_format"] = a.vis_format
    return kw


def _vis_ext(vis_format):
    if vis_format not in ("jpg", "png"):
        raise ValueError("vis_format must be jpg or png, not %r" % (vis_format,))
    return "." + vis_format


def _load_checkpoints(a):
    """-> (SMAP state dict, RefineNet state dict or None); FileNotFoundError with the reference's message."""
    if not os.path.exists(a.SMAP_path):
        raise FileNotFoundError("No such checkpoint of SMAP {}".format(a.SMAP_path))  # test.py:222
    sd = torch.load(a.SMAP_path, map_location="cpu")["model"]          # test.py:210-212
    rsd = None
    if a.RefineNet_path:
        if not os.path.exists(a.RefineNet_path):
            raise FileNotFoundError("No such RefineNet checkpoint of {}".format(a.RefineNet_path))  # test.py:216
        rsd = torch.load(a.RefineNet_path, map_location="cpu")         # test.py:214
    return sd, rsd


def _report(out, n, stats):
    print("Pairs writed to {} ({} images)".format(out, n))             # test.py:152
    if stats.get("saturation"):
        print("fp16: {} activation values exceeded +-65504 and were clamped; rerun with --precision bf16x3 (or bf16) "
              "for exact results".format(stats["saturation"]))


def _main_distributed(a):
    """main() under torchrun: one process per GPU, run_distributed; every rank returns 1 when any rank fails."""
    import traceback

    import torch.distributed as dist

    dist.init_process_group("gloo")
    rank = dist.get_rank()
    out = result_file_name(a.output_dir, a.test_mode, a.data_mode, a.json_name)
    try:
        err = None
        try:
            sd, rsd = _load_checkpoints(a)
            if rank == 0:
                os.makedirs(a.output_dir, exist_ok=True)
        except Exception as e:
            err = e
        _agree(err)
        stats = {}
        n = run_distributed(sd, a.dataset_path, out, rsd, a.batch_size, a.do_flip, a.dataset_name,
                            glob_order=bool(a.glob_order), precision=a.precision, stats=stats,
                            jpeg_colour=bool(a.jpeg_colour), **_vis_kwargs(a))
    except (FileNotFoundError, RankFailed) as e:
        print("rank {}: {}".format(rank, e), flush=True)
        return 1
    except Exception:
        print("rank {}: failed".format(rank), flush=True)
        traceback.print_exc()
        return 1
    finally:
        dist.destroy_process_group()
    if rank == 0:
        _report(out, n, stats)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
