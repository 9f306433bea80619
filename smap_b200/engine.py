"""Python host side of the hot path: a thin, torch-tensor-facing wrapper over the C ABI.

torch is plumbing only (device memory, streams); every kernel runs inside libsmap_b200.so."""
import ctypes
import os

import numpy as np
import torch

from . import _lib
from ._lib import MAXP, NC2D, NJ, NL, PREC_BF16, PREC_BF16X3, PREC_FP16, RECORD_BYTES, SCALE_LEN, SmapB200Error

RECORD_DTYPE = np.dtype([("pred3d", "<f8", (MAXP, NJ, 4)), ("root_depth", "<f8", (MAXP,)),
                         ("pred2d", "<f4", (MAXP, NJ, 4)), ("count", "<i4"), ("pad_", "<i4")])
assert RECORD_DTYPE.itemsize == RECORD_BYTES

# bf16x3: fp32-faithful (split-bf16 operands, 3 MMAs); fp16: the cost of bf16 with 4x finer rounding, range +-65504
# (Engine.saturation_count); bf16: the cost of fp16 with fp32's range and 8-bit mantissa
PRECISIONS = {"bf16x3": PREC_BF16X3, "fp16": PREC_FP16, "bf16": PREC_BF16}


def scale_row(scale):
    """dict (exps/stage3_root2/test.py:99-103 layout) -> float64[9]."""
    return np.array([scale["scale"], scale["img_width"], scale["img_height"], scale["net_width"],
                     scale["net_height"], scale["f_x"], scale["f_y"], scale["cx"], scale["cy"]], np.float64)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


TILE_TABLE_PATH = os.environ.get("SMAPB_TILE_TABLE") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "tiles", "h100.tsv")  # SMAPB_TILE_TABLE: another table (A/B of a re-tune)
_tile_table_loaded = False


def load_tile_table(path=TILE_TABLE_PATH):
    """Install the committed tile-shape table (process-wide, once): every process / rank then runs every layer with the
    same tile shape (BLOCK_N, variant), which makes results independent of the handle and of the rank.  Geometries the table does
    not cover are autotuned by the library (use smap_b200.dist.sync_tile_table to share rank 0's choices)."""
    global _tile_table_loaded
    if _tile_table_loaded or os.environ.get("SMAPB_NO_TILE_TABLE"):
        return 0
    _tile_table_loaded = True
    if not os.path.exists(path):
        return 0
    return _lib.load().smapb_set_tile_table(open(path, "rb").read())


def get_tile_table():
    """The process-wide tile table as text (committed table + whatever the autotuner added)."""
    lib = _lib.load()
    n = lib.smapb_get_tile_table(None, 0)
    buf = ctypes.create_string_buffer(n)
    lib.smapb_get_tile_table(buf, n)
    return buf.value.decode()


JPEG_SCANS = 1  # SMAPB_JPEG_SCANS
JPEG_COLOUR = 2  # SMAPB_JPEG_COLOUR
ENCODE_VIEW3D = 1  # SMAPB_ENCODE_VIEW3D


def _header_info(fn, data, *flags):
    """fn(data, nbytes, *flags, &h, &w, &orientation, &status), a header-only info entry point -> (status, h, w,
    orientation)."""
    h, w, o, st = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = fn(bytes(data), len(data), *flags, ctypes.byref(h), ctypes.byref(w), ctypes.byref(o), ctypes.byref(st))
    if rc != 0:
        raise SmapB200Error("%s failed (%d)" % (fn.__name__, rc))
    return st.value, h.value, w.value, o.value


def _jpeg_flags(scans, colour):
    return (JPEG_SCANS if scans else 0) | (JPEG_COLOUR if colour else 0)


def jpeg_info(data, scans=False, colour=False):
    """Header walk of one JPEG file on the host (no GPU): -> (status, h, w, orientation).  status 0 = the GPU decoder
    handles it and cv2.imread returns an [h, w, 3] image; otherwise one of SMAPB_JPEG_* (include/smap_b200.h).
    scans=True: the walk of Engine.decode_jpeg_ex, which also takes multi-scan sequential and progressive files;
    colour=True: it also takes CMYK, YCCK and RGB frames and every integral sampling (SMAPB_JPEG_COLOUR)."""
    return _header_info(_lib.load().smapb_jpeg_info_ex, data, _jpeg_flags(scans, colour))


def png_info(data):
    """Chunk walk of one PNG file on the host (no GPU): -> (status, h, w, orientation).  status 0 = the GPU decoder
    handles it and cv2.imread returns an [h, w, 3] image; otherwise one of SMAPB_JPEG_* (include/smap_b200.h)."""
    return _header_info(_lib.load().smapb_png_info, data)


class Engine:
    """One handle per (process, device).  in_h/in_w: network input size (multiples of 32)."""

    def __init__(self, device=0, max_batch=8, in_h=512, in_w=832, stream=None):
        """stream: None = every call runs on torch's current stream (the library bridges the legacy default stream to its
        own non-blocking stream); a torch.cuda.Stream = the handle's calls are issued on that stream and the caller orders
        it against other streams (pipelined use: several handles in flight, see EnginePool / bench.py)."""
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise SmapB200Error("smap_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        load_tile_table()
        self.device = torch.device("cuda", device)
        self.stream = stream
        self.world, self.rank = 1, 0
        self.max_batch, self.in_h, self.in_w = max_batch, in_h, in_w
        self.h, self.w = in_h // 4, in_w // 4
        hp = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            rc = self.lib.smapb_create(ctypes.byref(hp), device, max_batch, in_h, in_w)
        if rc != 0:
            raise SmapB200Error("smapb_create failed (%d): %s" % (rc, self.lib.smapb_last_error(None).decode()))
        self._h = hp
        self.precision = None

    def close(self):
        if getattr(self, "_h", None):
            self.lib.smapb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _st(self):
        return ctypes.c_void_p(self.stream.cuda_stream) if self.stream is not None else _stream()

    def _check(self, rc, what):
        if rc != 0:
            raise SmapB200Error("%s failed (%d): %s" % (what, rc, self.lib.smapb_last_error(self._h).decode()))

    # ---- weights ------------------------------------------------------------------------------
    def load_state_dict(self, sd, precision="bf16x3"):
        """sd: reference schema (model/smap.py, 1876 keys); tensors or arrays, any device."""
        for k, v in sd.items():
            if k.endswith("num_batches_tracked"):
                continue
            a = v.detach().cpu().float().contiguous().numpy() if torch.is_tensor(v) else np.ascontiguousarray(v, np.float32)
            shape = (ctypes.c_int64 * max(1, a.ndim))(*a.shape)
            self._check(self.lib.smapb_load_weight(self._h, k.encode(), a.ctypes.data_as(ctypes.c_void_p), shape, a.ndim),
                        "smapb_load_weight(%s)" % k)
        self._check(self.lib.smapb_finalize_weights(self._h, PRECISIONS[precision]), "smapb_finalize_weights")
        self.precision = precision

    # ---- backbone -----------------------------------------------------------------------------
    def forward(self, imgs):
        """imgs fp32 NCHW cuda [B,3,in_h,in_w] -> (hm2d [B,43,h,w], det_d [B,14,h,w], root_d [B,1,h,w])."""
        assert imgs.is_cuda and imgs.dtype == torch.float32 and imgs.shape[1:] == (3, self.in_h, self.in_w)
        imgs = imgs.contiguous()
        B = imgs.shape[0]
        hm = torch.empty(B, NC2D, self.h, self.w, device=imgs.device)
        dd = torch.empty(B, NL, self.h, self.w, device=imgs.device)
        rd = torch.empty(B, 1, self.h, self.w, device=imgs.device)
        self._check(self.lib.smapb_backbone_forward(self._h, _ptr(imgs), B, _ptr(hm), _ptr(dd), _ptr(rd), _stream()),
                    "smapb_backbone_forward")
        return hm, dd, rd

    def merge_scale(self, hm, hm_flip=None, do_scale=True):
        self._check(self.lib.smapb_merge_scale(self._h, _ptr(hm), _ptr(hm_flip), hm.shape[0], int(do_scale), _stream()),
                    "smapb_merge_scale")
        return hm

    # ---- association --------------------------------------------------------------------------
    def extract(self, hms):
        """hms fp32 cuda [B,43,h,w] (already /255,/127) -> peaks [B,15,128,3], pair scores [B,14,127,127]."""
        hms = hms.contiguous()
        B = hms.shape[0]
        peaks = torch.empty(B, NJ, MAXP + 1, 3, device=hms.device)
        scores = torch.empty(B, NL, MAXP, MAXP, device=hms.device)
        self._check(self.lib.smapb_assoc_extract(self._h, _ptr(hms), B, _ptr(peaks), _ptr(scores), _stream()),
                    "smapb_assoc_extract")
        return peaks, scores

    def connect(self, hms, rdepth, root_idx=2, dist_flag=True):
        """-> bodies [B,127,15,4] (x,y,0,score; heat-map px), counts int32 [B]; device tensors."""
        hms = hms.contiguous()
        rdepth = rdepth.contiguous()
        B = hms.shape[0]
        bodies = torch.empty(B, MAXP, NJ, 4, device=hms.device)
        counts = torch.empty(B, dtype=torch.int32, device=hms.device)
        self._check(self.lib.smapb_assoc_connect(self._h, _ptr(hms), _ptr(rdepth), B, root_idx, int(dist_flag),
                                                 _ptr(bodies), _ptr(counts), _stream()), "smapb_assoc_connect")
        return bodies, counts

    def lift(self, bodies, counts, det_d, root_d, scales):
        """scales: float64 cuda [B,9].  -> pred2d [B,127,15,4] f32, pred3d f64, root_depth [B,127] f64, counts."""
        B = bodies.shape[0]
        dev = bodies.device
        p2 = torch.empty(B, MAXP, NJ, 4, device=dev)
        p3 = torch.empty(B, MAXP, NJ, 4, device=dev, dtype=torch.float64)
        rdp = torch.empty(B, MAXP, device=dev, dtype=torch.float64)
        co = torch.empty(B, dtype=torch.int32, device=dev)
        self._check(self.lib.smapb_lift3d(self._h, _ptr(bodies.contiguous()), _ptr(counts), _ptr(det_d.contiguous()),
                                          _ptr(root_d.contiguous()), _ptr(scales.contiguous()), B, _ptr(p2), _ptr(p3),
                                          _ptr(rdp), _ptr(co), _stream()), "smapb_lift3d")
        return p2, p3, rdp, co

    def lift_gt(self, bodies, counts, det_d, root_d, scales, gt_roots, gt_counts):
        """Lift with ground truth (register_pred's matching branch, test_util.py:21-39).  gt_roots: float64 cuda [B,G,2]
        (GT root joints, network-input pixels), gt_counts: int32 cuda [B].  -> pred2d f64 [B,127,15,4], pred3d f64,
        root_depth f64 [B,127], counts int32 [B] (= gt_counts, or 0 for skipped frames); row g <-> GT person g."""
        B = bodies.shape[0]
        dev = bodies.device
        p2 = torch.empty(B, MAXP, NJ, 4, device=dev, dtype=torch.float64)
        p3 = torch.empty(B, MAXP, NJ, 4, device=dev, dtype=torch.float64)
        rdp = torch.empty(B, MAXP, device=dev, dtype=torch.float64)
        co = torch.empty(B, dtype=torch.int32, device=dev)
        gt_roots = gt_roots.to(torch.float64).contiguous()
        assert gt_roots.dim() == 3 and gt_roots.shape[0] == B and gt_roots.shape[2] == 2
        self._check(self.lib.smapb_lift3d_gt(self._h, _ptr(bodies.contiguous()), _ptr(counts), _ptr(det_d.contiguous()),
                                             _ptr(root_d.contiguous()), _ptr(scales.contiguous()), _ptr(gt_roots),
                                             _ptr(gt_counts.to(torch.int32).contiguous()), gt_roots.shape[1], B, _ptr(p2), _ptr(p3),
                                             _ptr(rdp), _ptr(co), self._st()), "smapb_lift3d_gt")
        return p2, p3, rdp, co

    # ---- image decoding ------------------------------------------------------------------------
    def _decode(self, files, info, fn, *flags):
        """Output tensors sized by info(file) -> (status, h, w, orientation), then one batch call fn(handle, n, files,
        sizes, outputs, *flags, status, stream) -> per file the tensor, or None where the status is not 0."""
        n = len(files)
        out = [None] * n
        if n == 0:
            return out
        ptrs = (ctypes.c_void_p * n)()
        for i, f in enumerate(files):
            st, h, w = info(f)[:3]
            if st == 0:
                out[i] = torch.empty(h, w, 3, dtype=torch.uint8, device=self.device)
                ptrs[i] = out[i].data_ptr()
        data = (ctypes.c_char_p * n)(*files)
        sizes = (ctypes.c_int64 * n)(*[len(f) for f in files])
        status = (ctypes.c_int * n)()
        self._check(fn(self._h, n, data, sizes, ptrs, *flags, status, self._st()), fn.__name__)
        return [o if status[i] == 0 else None for i, o in enumerate(out)]

    def decode_jpeg(self, files):
        """files: list of bytes (whole JPEG files) -> list with, per file, a CUDA uint8 BGR [H,W,3] tensor equal to
        cv2.imdecode(file, IMREAD_COLOR), or None when the file is not one the GPU decoder handles (cv2 must read it)."""
        return self._decode(files, jpeg_info, self.lib.smapb_decode_jpeg)

    def decode_jpeg_ex(self, files, scans=True, colour=False):
        """decode_jpeg for a batch that may also hold progressive Huffman files and sequential files with several scans
        (smapb_decode_jpeg_ex with SMAPB_JPEG_SCANS; scans=False and colour=False is decode_jpeg), and with colour=True
        CMYK, YCCK and RGB frames and every integral sampling (SMAPB_JPEG_COLOUR: 4:1:1, 4:1:0, factors of 3, chroma
        finer than luma).  -> per file a CUDA uint8 BGR [H,W,3] tensor equal to cv2.imdecode(file, IMREAD_COLOR), or None
        (cv2 must read it).  Progressive files decode their AC refinement scans sequentially within each restart segment
        (one warp per segment, the batch's images side by side), so a batch takes about as long as its slowest image;
        run_inference sends the JPEGs decode_jpeg refuses here."""
        return self._decode(files, lambda f: jpeg_info(f, scans, colour), self.lib.smapb_decode_jpeg_ex,
                            _jpeg_flags(scans, colour))

    def decode_png(self, files):
        """files: list of bytes (whole PNG files) -> list with, per file, a CUDA uint8 BGR [H,W,3] tensor equal to
        cv2.imdecode(file, IMREAD_COLOR), or None when the file is not one the GPU decoder handles (cv2 must read it)."""
        return self._decode(files, png_info, self.lib.smapb_decode_png)

    def png_stats(self):
        """Inflate counters of the last decode_png call (smapb_png_inflate_stats): dict with candidates, false_positives,
        confirmed (chained blocks found by the block finder) and serial (chained blocks the serial walk handled)."""
        v = (ctypes.c_int64 * 4)()
        self._check(self.lib.smapb_png_inflate_stats(self._h, v), "smapb_png_inflate_stats")
        return dict(zip(("candidates", "false_positives", "confirmed", "serial"), list(v)))

    # ---- image encoding --------------------------------------------------------------------------
    def encode_jpeg(self, frames, quality=95, records=None, scales=None, view3d=False):
        """frames: list of uint8 BGR [H,W,3] tensors (cuda, or cpu / numpy arrays, which are uploaded) -> list of bytes, per
        frame what cv2.imencode(".jpg", frame, [IMWRITE_JPEG_QUALITY, quality]) writes.  records (uint8 [n, RECORD_BYTES],
        as infer_device returns them) with scales (float64 [n, 9], the frames' scale rows from preprocess): each frame is
        encoded with its skeletons drawn over it (smapb_encode_jpeg, include/smap_b200.h).  view3d (records required):
        each H x W frame is encoded as an H x (W + H) composite, the drawn frame and an H x H panel of its 3D skeletons
        (smapb_encode_jpeg_ex with SMAPB_ENCODE_VIEW3D; oracle/view3d_numpy.py).  The frames are not modified."""
        a = self._encode_args("encode_jpeg", frames, records, scales, view3d)
        if a is None:
            return []
        n, ptrs, hs, ws, rec, sc, sizes = a
        if view3d:
            self._check(self.lib.smapb_encode_jpeg_ex(self._h, n, ptrs, hs, ws, int(quality), _ptr(rec), _ptr(sc), ENCODE_VIEW3D,
                                                      sizes, self._st()), "smapb_encode_jpeg_ex")
        else:
            self._check(self.lib.smapb_encode_jpeg(self._h, n, ptrs, hs, ws, int(quality), _ptr(rec), _ptr(sc), sizes,
                                                   self._st()), "smapb_encode_jpeg")
        return self._encoded(self.lib.smapb_encoded_jpeg, "smapb_encoded_jpeg", sizes)

    def encode_png(self, frames, records=None, scales=None, view3d=False):
        """As encode_jpeg, but lossless: per frame (or composite) what cv2.imencode(".png", frame) writes
        (smapb_encode_png, include/smap_b200.h; oracle/png_encode_numpy.py)."""
        a = self._encode_args("encode_png", frames, records, scales, view3d)
        if a is None:
            return []
        n, ptrs, hs, ws, rec, sc, sizes = a
        self._check(self.lib.smapb_encode_png(self._h, n, ptrs, hs, ws, _ptr(rec), _ptr(sc), ENCODE_VIEW3D if view3d else 0,
                                              sizes, self._st()), "smapb_encode_png")
        return self._encoded(self.lib.smapb_encoded_png, "smapb_encoded_png", sizes)

    def _encode_args(self, name, frames, records, scales, view3d):
        """The encoders' arguments: frames uploaded, records and scales checked -> (n, frame pointers, heights, widths,
        records, scales, sizes), or None for no frames.  The device copies live as long as the returned tuple."""
        n = len(frames)
        if view3d and records is None:
            raise ValueError("%s: view3d needs records and scales" % name)
        if n == 0:
            return None
        if (records is None) != (scales is None):
            raise ValueError("%s: records and scales go together" % name)
        dev = []
        for f in frames:
            if not torch.is_tensor(f):
                f = torch.from_numpy(np.ascontiguousarray(f))
            if f.dtype != torch.uint8 or f.dim() != 3 or f.shape[2] != 3:
                raise ValueError("%s: uint8 BGR [H,W,3] frames expected" % name)
            dev.append(f.to(self.device).contiguous())
        ptrs = (ctypes.c_void_p * n)(*[f.data_ptr() for f in dev])
        ptrs._frames = dev  # keeps the device copies alive with the pointer array
        hs = (ctypes.c_int * n)(*[f.shape[0] for f in dev])
        ws = (ctypes.c_int * n)(*[f.shape[1] for f in dev])
        rec = sc = None
        if records is not None:
            rec = records.to(self.device).contiguous()
            sc = torch.as_tensor(scales, dtype=torch.float64).to(self.device).contiguous()
            if rec.dtype != torch.uint8 or tuple(rec.shape) != (n, RECORD_BYTES) or tuple(sc.shape) != (n, SCALE_LEN):
                raise ValueError("%s: records uint8 [n, %d] and scales float64 [n, %d] expected" % (name, RECORD_BYTES, SCALE_LEN))
        return n, ptrs, hs, ws, rec, sc, (ctypes.c_int64 * n)()

    def _encoded(self, get, name, sizes):
        out = []
        for i in range(len(sizes)):
            p = ctypes.POINTER(ctypes.c_uint8)()
            self._check(get(self._h, i, ctypes.byref(p), None), name)
            out.append(ctypes.string_at(p, sizes[i]))
        return out

    # ---- pre-processing ------------------------------------------------------------------------
    def preprocess(self, images, out=None):
        """images: list of uint8 BGR [H,W,3] tensors (cuda or cpu; numpy arrays are taken as host images) ->
        (imgs fp32 cuda [B,3,in_h,in_w], scales float64 cpu [B,9]); dataset/custom_dataset.py:27-68 + test.py:99-103."""
        B = len(images)
        dev = self.device
        if out is None:
            out = torch.empty(B, 3, self.in_h, self.in_w, device=dev)
        scales = np.zeros((B, 9), np.float64)
        keep = []
        for b, im in enumerate(images):
            if not torch.is_tensor(im):
                im = torch.from_numpy(np.ascontiguousarray(im))
            assert im.dtype == torch.uint8 and im.dim() == 3 and im.shape[2] == 3, "uint8 BGR [H,W,3] expected"
            im = im.contiguous()
            keep.append(im)
            row = scales[b].ctypes.data_as(ctypes.POINTER(ctypes.c_double))
            fn = self.lib.smapb_preprocess if im.is_cuda else self.lib.smapb_preprocess_host
            self._check(fn(self._h, _ptr(im), im.shape[0], im.shape[1], ctypes.c_void_p(out[b].data_ptr()), row, _stream()),
                        "smapb_preprocess")
        if any(not im.is_cuda for im in keep):
            torch.cuda.current_stream().synchronize()  # host images must outlive their asynchronous upload
        return out, torch.from_numpy(scales)

    # ---- RefineNet (optional post-processing) ---------------------------------------------------
    def load_refine_state_dict(self, sd):
        """sd: state dict of the reference model/refinenet.py RefineNet (block.layerN...)."""
        for k, v in sd.items():
            if k.endswith("num_batches_tracked"):
                continue
            a = v.detach().cpu().float().contiguous().numpy() if torch.is_tensor(v) else np.ascontiguousarray(v, np.float32)
            shape = (ctypes.c_int64 * max(1, a.ndim))(*a.shape)
            self._check(self.lib.smapb_refine_load_weight(self._h, k.encode(), a.ctypes.data_as(ctypes.c_void_p), shape, a.ndim),
                        "smapb_refine_load_weight(%s)" % k)
        self._check(self.lib.smapb_refine_finalize(self._h), "smapb_refine_finalize")

    def refine_mlp(self, inp):
        """inp fp32 cuda [n,75] -> fp32 cuda [n,45] (refine_model(inp), model/refinenet.py:19-26)."""
        inp = inp.contiguous()
        out = torch.empty(inp.shape[0], 45, device=inp.device)
        self._check(self.lib.smapb_refine_mlp(self._h, _ptr(inp), inp.shape[0], _ptr(out), _stream()), "smapb_refine_mlp")
        return out

    def refine(self, pred2d, pred3d, counts, root_idx=2):
        """outputs of lift() -> refined fp64 cuda [B,127,15,4] (lift_and_refine_3d_pose, test_util.py:102-131); rows
        >= counts[b] are zero."""
        out = torch.zeros_like(pred3d)
        self._check(self.lib.smapb_refine3d(self._h, _ptr(pred2d.contiguous()), _ptr(pred3d.contiguous()), _ptr(counts),
                                            pred3d.shape[0], root_idx, _ptr(out), _stream()), "smapb_refine3d")
        return out

    def set_refine(self, enable=True):
        """infer_device / infer_host / submit_host store the refined poses in the records' pred3d field."""
        self._check(self.lib.smapb_set_refine(self._h, int(bool(enable))), "smapb_set_refine")

    # ---- whole path ---------------------------------------------------------------------------
    def infer_device(self, imgs, scales, do_flip=False, out=None, gather=False, defer=False):
        """imgs cuda fp32 [B,3,H,W], scales cuda f64 [B,9] -> records uint8 cuda [B, RECORD_BYTES]; gather=True (after
        init_comm): [world*B, RECORD_BYTES], all ranks' records in rank order, exchanged by ONE ncclAllGather on the same
        stream (inside the same CUDA graph).  defer=True (with gather): the exchange runs on the handle's gather stream and
        `out` is valid after gather_sync() - the compute stream never waits for peers (smapb_infer_device_gather_async).
        With an engine-owned stream the call is asynchronous with respect to torch's current stream: pass `out`
        (preallocated) and order the streams yourself."""
        B = imgs.shape[0]
        n = B * (self.world if gather else 1)
        if out is None:
            out = torch.empty(n, RECORD_BYTES, dtype=torch.uint8, device=imgs.device)
            if self.stream is not None:
                out.record_stream(self.stream)
        assert out.shape[0] == n and out.is_contiguous()
        fn = (self.lib.smapb_infer_device_gather_async if defer else self.lib.smapb_infer_device_gather) if gather \
            else self.lib.smapb_infer_device
        self._check(fn(self._h, _ptr(imgs.contiguous()), _ptr(scales.contiguous()), B, int(do_flip), _ptr(out), self._st()),
                    "smapb_infer_device")
        return out

    def gather_sync(self):
        """Order this engine's stream (or torch's current stream) after every outstanding deferred exchange."""
        self._check(self.lib.smapb_gather_sync(self._h, self._st()), "smapb_gather_sync")

    # ---- multi-GPU ------------------------------------------------------------------------------
    def init_comm(self, group=None):
        """Collective over the torch.distributed group: create this handle's own NCCL communicator (rank 0 makes the
        ncclUniqueId, torch.distributed only ships those 128 bytes).  Engines of a rank must call this in the same order
        on every rank."""
        import torch.distributed as dist

        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        uid = (ctypes.c_char * 128)()
        if self.rank == 0:
            rc = self.lib.smapb_comm_unique_id(uid)
            if rc != 0:
                raise SmapB200Error("smapb_comm_unique_id failed (%d): NCCL not loadable" % rc)
        box = [bytes(uid.raw)]
        dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        uid = (ctypes.c_char * 128).from_buffer_copy(box[0])
        with torch.cuda.device(self.device):
            self._check(self.lib.smapb_comm_create(self._h, uid, self.rank, self.world), "smapb_comm_create")

    def attach_torch_comm(self, group=None):
        """Borrow torch.distributed's own ncclComm_t (ProcessGroupNCCL._comm_ptr) instead of creating one."""
        import torch.distributed as dist

        pg = group if group is not None else dist.distributed_c10d._get_default_group()
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        backend = pg._get_backend(self.device)
        backend.eager_connect_single_device(self.device) if not backend._is_initialized() else None
        ptr = backend._comm_ptr()
        self._check(self.lib.smapb_comm_attach(self._h, ctypes.c_void_p(ptr), self.rank, self.world), "smapb_comm_attach")

    def allgather(self, rec, out=None):
        """rec uint8 cuda [B, RECORD_BYTES] -> [world*B, RECORD_BYTES] (smapb_allgather_records on this handle's comm)."""
        B = rec.shape[0]
        if out is None:
            out = torch.empty(self.world * B, RECORD_BYTES, dtype=torch.uint8, device=rec.device)
        self._check(self.lib.smapb_allgather_records(self._h, None, _ptr(rec.contiguous()), _ptr(out), B, self._st()),
                    "smapb_allgather_records")
        return out

    def infer_host(self, imgs, scales, do_flip=False, out=None):
        """Host buffers in, host records out (synchronous).  imgs: CPU fp32 tensor (pinned preferred) [B,3,H,W];
        scales: CPU float64 [B,9].  Returns a numpy structured array of RECORD_DTYPE [B]."""
        assert not imgs.is_cuda and imgs.dtype == torch.float32
        B = imgs.shape[0]
        if out is None:
            out = torch.empty(B, RECORD_BYTES, dtype=torch.uint8).pin_memory()
        scales = torch.as_tensor(scales, dtype=torch.float64).contiguous()
        self._check(self.lib.smapb_infer_host(self._h, _ptr(imgs.contiguous()), _ptr(scales), B, int(do_flip),
                                              _ptr(out), _stream()), "smapb_infer_host")
        return out.numpy().view(RECORD_DTYPE).reshape(B)

    def submit_host(self, slot, imgs, scales, out, do_flip=False, gather=False):
        """Pipelined infer_host: enqueue one batch on slot 0/1 and return immediately (see smapb_submit_host).
        imgs: pinned CPU fp32 [B,3,H,W]; scales: pinned CPU float64 [B,9]; out: pinned CPU uint8 [B, RECORD_BYTES]
        (gather=True: [world*B, RECORD_BYTES] - the records are all-gathered on the device before the single D2H)."""
        assert not imgs.is_cuda and imgs.dtype == torch.float32 and imgs.is_contiguous()
        assert scales.dtype == torch.float64 and out.dtype == torch.uint8
        assert out.shape[0] == imgs.shape[0] * (self.world if gather else 1)
        fn = self.lib.smapb_submit_host_gather if gather else self.lib.smapb_submit_host
        self._check(fn(self._h, slot, _ptr(imgs), _ptr(scales), imgs.shape[0], int(do_flip), _ptr(out)), "smapb_submit_host")

    def wait(self, slot):
        self._check(self.lib.smapb_wait(self._h, slot), "smapb_wait")

    # ---- introspection ------------------------------------------------------------------------
    def launch_count(self):
        return int(self.lib.smapb_launch_count(self._h))

    def saturation_count(self, reset=False):
        """fp16 precision: activation elements clamped to +-65504 since creation (or the last reset=True); synchronises the
        device.  Nonzero means some outputs are not the model's: use precision "bf16x3" (or "bf16") for such inputs."""
        n = self.lib.smapb_saturation_count(self._h, int(bool(reset)))
        if n < 0:
            raise SmapB200Error("smapb_saturation_count failed (%d): %s" % (n, self.lib.smapb_last_error(self._h).decode()))
        return int(n)

    def profile_begin(self):
        self._check(self.lib.smapb_profile_begin(self._h), "smapb_profile_begin")

    def profile_end(self, csv_path=None):
        """-> dict kind -> (ms, launches); kinds: conv, stem, elementwise, assoc, lift."""
        ms = (ctypes.c_double * 6)()
        n = (ctypes.c_int * 6)()
        self._check(self.lib.smapb_profile_end(self._h, ms, n, csv_path.encode() if csv_path else None), "smapb_profile_end")
        names = ["conv", "stem", "elementwise", "assoc", "lift", "other"]
        return {names[i]: (ms[i], n[i]) for i in range(6)}

    def plan_info(self, B):
        n = ctypes.c_int()
        f = ctypes.c_double()
        self._check(self.lib.smapb_plan_info(self._h, B, ctypes.byref(n), ctypes.byref(f)), "smapb_plan_info")
        return n.value, f.value

    def conv_test(self, x, w, bias, res=None, stride=1, relu=True, precision="bf16x3", time_it=False, post1=None,
                  post2=None, in2=None, stride2=1, up=None, out_f32=False, launch=None):
        """One convolution through the tensor-core path (smapb_conv_test).  x fp32 NHWC cuda [B,H,W,Cin]; w
        [Cout,Cin+Cin2,k,k], Cin2 the channels of in2 (fp32 NHWC, the K-concatenated 1x1 input of a fused pair, with
        stride2); up fp32 NHWC at half the output size (fused bilinear residual); out_f32: fp32 output as the head convs
        store it.  launch: a dict that receives block_n, tw, flat and ring of the launch.  Returns y fp32 NHWC (and ms)."""
        B, H, W, Cin = x.shape
        Cout, _, k, _ = w.shape
        H2, W2, Cin2 = in2.shape[1:] if in2 is not None else (0, 0, 0)
        pad = k // 2
        Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        y = torch.empty(B, Ho, Wo, Cout, device=x.device)
        ms = ctypes.c_float(0)
        ran = (ctypes.c_int * 4)()
        args = [t.contiguous() if t is not None else None for t in (x, w, bias, res, post1, post2, in2, up)]
        self._check(self.lib.smapb_conv_test(self._h, *[_ptr(t) for t in args], B, H, W, Cin, Cout, k, stride, H2, W2,
                                             Cin2, stride2, int(relu), int(out_f32),
                                             PRECISIONS[precision], _ptr(y), ran, ctypes.byref(ms) if time_it else None,
                                             _stream()), "smapb_conv_test")
        if launch is not None:
            launch.update(block_n=ran[0], tw=ran[1], flat=bool(ran[2]), ring=ran[3])
        return (y, ms.value) if time_it else y


def records_to_numpy(rec):
    """uint8 cuda/cpu tensor [B, RECORD_BYTES] -> numpy structured array [B]."""
    return rec.cpu().numpy().view(RECORD_DTYPE).reshape(rec.shape[0])


class EnginePool:
    """N independent handles on one GPU (each with its own workspace, plan and streams), used round-robin so that N
    batches are in flight: the tail of one batch's kernels (partial last waves) overlaps the other batch's kernels and
    the H2D of the next batch overlaps compute.  Two handles keep two batches in flight (bench.py --engines)."""

    def __init__(self, n=2, device=0, max_batch=8, in_h=512, in_w=832):
        self.engines = [Engine(device, max_batch, in_h, in_w) for _ in range(n)]
        self._next = 0
        self._tickets = {}

    def load_state_dict(self, sd, precision="bf16x3"):
        for e in self.engines:
            e.load_state_dict(sd, precision)

    def load_refine_state_dict(self, sd, enable=True):
        """RefineNet weights for every handle; enable=True makes the records carry the refined poses."""
        for e in self.engines:
            e.load_refine_state_dict(sd)
            e.set_refine(enable)

    def submit(self, imgs, scales, out, do_flip=False):
        """Enqueue one host batch (pinned tensors, see Engine.submit_host); returns a ticket for result()."""
        t = self._next
        self._next += 1
        n = len(self.engines)
        e, slot = self.engines[t % n], (t // n) % 2
        prev = t - 2 * n
        if prev in self._tickets and not self._tickets[prev][3]:
            # the slot is about to be reused: wait for its previous occupant (its records stay in the caller's `out`
            # buffer, so result(prev) still works afterwards)
            pe, pslot, pout, _ = self._tickets[prev]
            pe.wait(pslot)
            self._tickets[prev] = (pe, pslot, pout, True)
        e.submit_host(slot, imgs, scales, out, do_flip)
        self._tickets[t] = (e, slot, out, False)
        return t

    def result(self, ticket):
        """Block until the batch is done; returns its records as a numpy structured array."""
        if ticket not in self._tickets:
            raise SmapB200Error("EnginePool.result: unknown or already collected ticket %r" % (ticket,))
        e, slot, out, done = self._tickets.pop(ticket)
        if not done:
            e.wait(slot)
        return out.numpy().view(RECORD_DTYPE).reshape(out.shape[0])

    def close(self):
        for e in self.engines:
            e.close()
