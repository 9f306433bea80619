"""`run_inference` mode of the reference CLI (exps/stage3_root2/test.py:154-225 with `-t run_inference`) on the fused
path: images on disk -> result JSON.

    python -m smap_b200.run_inference -p SMAP.pth [-rp RefineNet.pth] --dataset_path DIR --batch_size 8 --do_flip 1 \
        [--json_name SUFFIX] [--output_dir OUT] [--dataset_name CMU] [--precision {bf16x3,fp16,bf16}] [--jpeg_colour 1]

Same flags and the same output file name / schema as the reference ('{OUT}/stage3_root2_run_inference_{data_mode}_{suffix}.json',
test.py:147-152).  Differences, both deliberate: images are visited in sorted path order unless --glob_order 1 (the
reference uses glob order, dataset/custom_dataset.py:16-18).  Decoding, resize, letterbox, normalisation, backbone,
association, lift, RefineNet and the JSON text are produced by libsmap_b200.so: .jpg/.jpeg and .png files the GPU decoders
support are decoded on the GPU (byte-identical to cv2.imread), every other file by cv2.imread as in the reference.  Baseline
JPEGs go through Engine.decode_jpeg; progressive and multi-scan JPEGs through Engine.decode_jpeg_ex, in a batch of their own,
which with --jpeg_colour 1 also takes CMYK, YCCK and RGB JPEGs and every integral sampling (4:1:1, 4:1:0, ...).
"""
import argparse
import functools
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


def run(smap_state_dict, dataset_path, output_file, refine_state_dict=None, batch_size=8, do_flip=False, dataset_name="CMU",
        device=0, in_h=512, in_w=832, imread=None, glob_order=False, precision="bf16x3", stats=None, jpeg_colour=False):
    """-> number of images processed.  imread(path) -> uint8 BGR [H,W,3], used for every file; by default .jpg/.jpeg
    and .png files are decoded on the GPU (Engine.decode_jpeg, then Engine.decode_jpeg_ex for the progressive and
    multi-scan JPEGs decode_jpeg leaves, and Engine.decode_png; byte-identical to cv2.imread) and the
    files they do not handle, as every other file, go through cv2.imread(path, IMREAD_COLOR).  jpeg_colour=True: CMYK,
    YCCK and RGB JPEGs and every integral sampling are decoded on the GPU too (Engine.decode_jpeg_ex(colour=True));
    off by default, so those files keep going to cv2.imread.  precision: one of engine.PRECISIONS.  stats (a dict,
    optional) receives "saturation": the fp16 clamp count."""
    if precision not in PRECISIONS:
        raise ValueError("unknown precision %r (choose from %s)" % (precision, ", ".join(PRECISIONS)))
    gpu_decode = imread is None
    if imread is None:
        import cv2

        def imread(p):
            im = cv2.imread(p, cv2.IMREAD_COLOR)
            if im is None:
                raise RuntimeError("cannot read image " + p)
            return im

    eng = Engine(device, max_batch=batch_size, in_h=in_h, in_w=in_w)
    try:
        eng.load_state_dict(smap_state_dict, precision)
        if refine_state_dict is not None:
            eng.load_refine_state_dict(refine_state_dict)
            eng.set_refine(True)
        paths = list_images(dataset_path, glob_order)
        read = functools.partial(read_frames, jpeg_colour=True) if jpeg_colour else read_frames
        host = torch.empty(batch_size, RECORD_BYTES, dtype=torch.uint8).pin_memory()
        with ResultWriter(output_file, dataset_name) as w:
            for lo in range(0, len(paths), batch_size):
                chunk = paths[lo:lo + batch_size]
                frames = read(eng, chunk, imread) if gpu_decode else [imread(p) for p in chunk]
                frames = [f if torch.is_tensor(f) else torch.from_numpy(np.ascontiguousarray(f)) for f in frames]
                imgs, scales = eng.preprocess(frames)
                rec = eng.infer_device(imgs, scales.to(imgs.device), do_flip=bool(do_flip))
                host[:len(chunk)].copy_(rec)
                torch.cuda.current_stream().synchronize()
                w.append(host[:len(chunk)], [image_name(p, dataset_path) for p in chunk])
        if stats is not None:
            stats["saturation"] = eng.saturation_count()
        return len(paths)
    finally:
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
    a = ap.parse_args(argv)
    if not os.path.exists(a.SMAP_path):
        print("No such checkpoint of SMAP {}".format(a.SMAP_path))  # test.py:222
        return 1
    sd = torch.load(a.SMAP_path, map_location="cpu")["model"]          # test.py:210-212
    rsd = None
    if a.RefineNet_path:
        if not os.path.exists(a.RefineNet_path):
            print("No such RefineNet checkpoint of {}".format(a.RefineNet_path))  # test.py:216
            return 1
        rsd = torch.load(a.RefineNet_path, map_location="cpu")         # test.py:214
    os.makedirs(a.output_dir, exist_ok=True)
    out = result_file_name(a.output_dir, a.test_mode, a.data_mode, a.json_name)
    stats = {}
    n = run(sd, a.dataset_path, out, rsd, a.batch_size, a.do_flip, a.dataset_name, glob_order=bool(a.glob_order),
            precision=a.precision, stats=stats, jpeg_colour=bool(a.jpeg_colour))
    print("Pairs writed to {} ({} images)".format(out, n))             # test.py:152
    if stats.get("saturation"):
        print("fp16: {} activation values exceeded +-65504 and were clamped; rerun with --precision bf16x3 (or bf16) "
              "for exact results".format(stats["saturation"]))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
