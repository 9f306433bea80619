/*
 * smap_b200 - C ABI of the H100-native SMAP inference hot path.
 *
 * Plain C: opaque handle, raw pointers, sizes, int error codes (0 = ok, < 0 = error; the text is
 * available from smapb_last_error()).  Nothing throws across this boundary, no torch types appear in
 * it.  All *_dev pointers are device pointers on the handle's device, caller-owned; the handle owns
 * its workspace (no per-call cudaMalloc).  Calls are stream-ordered on `stream` (a cudaStream_t passed
 * as void*; NULL = legacy default stream) and do NOT synchronise unless stated.
 *
 * Each entry point names the reference interface it replaces (paths relative to zju3dv/SMAP).
 */
#ifndef SMAP_B200_H
#define SMAP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct smapb_handle smapb_handle;

#define SMAPB_NJ 15        /* key points,            extensions/association.cpp:18 */
#define SMAPB_NL 14        /* limbs,                 extensions/association.cpp:19 */
#define SMAPB_MAXP 127     /* max peaks per channel, extensions/association.cpp:20 */
#define SMAPB_NC2D 43      /* 2D head channels,      model/smap.py:320 */
#define SMAPB_SCALE_LEN 9  /* scale,img_w,img_h,net_w,net_h,f_x,f_y,cx,cy (exps/stage3_root2/test.py:99-103) */

/* precision of the tensor-core convolutions */
#define SMAPB_PREC_BF16X3 3 /* split-bf16 (hi+lo) operands, 3 MMAs per product, fp32 accumulate: fp32-faithful */
#define SMAPB_PREC_BF16 1   /* single bf16 operands (fast, ~1e-2 relative; NOT parity grade) */
/* single fp16 operands and activations: the cost of SMAPB_PREC_BF16 (same bytes, same MMA rate) with a 10-bit mantissa
 * (4x finer rounding; the operand precision of cuDNN's TF32 convolutions).  fp16 is finite only up to 65504: folded weights
 * beyond it make smapb_finalize_weights fail, and activations beyond it are clamped to +-65504 and counted
 * (smapb_saturation_count). */
#define SMAPB_PREC_FP16 16

/* ---- lifetime -------------------------------------------------------------------------------- */
/* Replaces: per-call ArrayGpu<T> scratch (extensions/arraygpu.hpp:62-77, re-created on every
 * extract(), extensions/association.cpp:47-63) and SMAP(cfg).to('cuda') (exps/stage3_root2/test.py:190-192).
 * in_h/in_w: network input size (multiples of 32); heat-maps are in_h/4 x in_w/4. */
int smapb_create(smapb_handle** out, int device, int max_batch, int in_h, int in_w);
void smapb_destroy(smapb_handle* h);
const char* smapb_last_error(const smapb_handle* h); /* never NULL; h may be NULL for create errors */
int smapb_version(void);

/* ---- weights (model/smap.py state-dict schema, 268 conv_bn_relu units x 7 tensors) ------------ */
/* Replaces: model.load_state_dict(sd) (exps/stage3_root2/test.py:210-212).  `key` is the reference
 * key ("stage0.downsample.layer1.0.conv_bn_relu1.conv.weight", "top.conv.bn.running_var", ...),
 * `host` fp32 host data, copied.  num_batches_tracked keys are accepted and ignored. */
int smapb_load_weight(smapb_handle* h, const char* key, const float* host, const int64_t* shape, int ndim);
/* BN folding (model/smap.py:23, eps 1e-5), NHWC/K-major repack, hi/lo split, TMA descriptors,
 * execution plan.  precision: SMAPB_PREC_*.  Must be called once after all weights are loaded. */
int smapb_finalize_weights(smapb_handle* h, int precision);

/* ---- pre-processing (the step in front of the backbone) ------------------------------------------------------ */
/* Replaces: CustomDataset.__getitem__ after cv2.imread (dataset/custom_dataset.py:27-68): scale = min(net_w/W, net_h/H),
 * cv2.resize(img, (0,0), fx=scale, fy=scale) (8-bit INTER_LINEAR, bit-exact incl. the 1/2-scale INTER_AREA reroute and
 * its partial blocks at an odd last column or row), gray-128 letterbox to net_w x net_h, torchvision ToTensor +
 * Normalize(cfg.INPUT.MEANS, cfg.INPUT.STDS).  img_w and img_h: 1 to 16384.  Returns -1 (smapb_last_error names the
 * geometry) where cv2.resize raises: when rint(img_w * scale) or rint(img_h * scale) is 0, e.g. 16x16384 into 832x512.
 * bgr_dev: uint8 [img_h, img_w, 3] (BGR, as cv2.imread returns); out_nchw_dev: fp32 [3, in_h, in_w] - one image slot of the
 * batch handed to smapb_backbone_forward / smapb_infer_device.  scale_row_host (may be NULL): the image's 9 scale values
 * in SMAPB_SCALE_LEN order, including the default intrinsics of exps/stage3_root2/test.py:99-103. */
int smapb_preprocess(smapb_handle* h, const uint8_t* bgr_dev, int img_h, int img_w, float* out_nchw_dev, double* scale_row_host,
                     void* stream);
/* Same with the image in host memory (pinned for an asynchronous copy): uploads the uint8 pixels - 4x fewer bytes than
 * the fp32 tensor the reference's loader ships - into the handle's staging buffer first. */
int smapb_preprocess_host(smapb_handle* h, const uint8_t* bgr_host, int img_h, int img_w, float* out_nchw_dev,
                          double* scale_row_host, void* stream);

/* ---- JPEG decoding (the step in front of pre-processing) ------------------------------------------------------------- */
/* Replaces: cv2.imread(path, IMREAD_COLOR) (dataset/custom_dataset.py:27) for the JPEGs it can decode, byte for byte:
 * baseline / extended-sequential Huffman (SOF0/SOF1), 8-bit samples, 8- or 16-bit DQT, any DHT (optimised tables too),
 * DRI restart intervals, one interleaved scan of every component, grayscale (replicated to BGR) or 3 components libjpeg
 * treats as YCbCr, luma sampling H, V in {1, 2} with chroma 1x1 (4:4:4, 4:2:2, 4:4:0, 4:2:0), EXIF orientation 1..8 applied
 * as cv2 applies it, up to SMAPB_JPEG_MAX_PIXELS.  Everything else (progressive, arithmetic, 12-bit, lossless, CMYK, RGB,
 * other sampling, several scans, non-JPEG data, truncated or corrupt data) gets a status != SMAPB_JPEG_OK and is meant for
 * cv2.imread. */
#define SMAPB_JPEG_OK 0
#define SMAPB_JPEG_UNSUPPORTED 1 /* a JPEG (or a block of one) this decoder does not handle */
#define SMAPB_JPEG_MALFORMED 2   /* not a JPEG, or a header that does not parse */
#define SMAPB_JPEG_CORRUPT 3     /* entropy-coded data that does not decode to the frame's blocks */
#define SMAPB_JPEG_TOO_LARGE 4   /* over SMAPB_JPEG_MAX_PIXELS */
#define SMAPB_JPEG_MAX_PIXELS (1 << 26)
/* Host only (no GPU work): header walk of one file.  *status = SMAPB_JPEG_*; when it is SMAPB_JPEG_OK, *h x *w is the shape
 * cv2.imread returns (after the EXIF orientation) and *orientation the EXIF value (1 without one); zeros otherwise.
 * Returns 0, or -1 for a NULL status. */
int smapb_jpeg_info(const uint8_t* data, int64_t nbytes, int* h, int* w, int* orientation, int* status);
/* Decodes n files (host memory) into bgr_dev[i]: uint8 [h, w, 3] BGR as smapb_jpeg_info reports the shape, which
 * smapb_preprocess consumes.  bgr_dev[i] may be NULL only for files smapb_jpeg_info does not accept.  status_host[i]
 * (SMAPB_JPEG_*) says whether bgr_dev[i] holds the image; the header status can turn into SMAPB_JPEG_CORRUPT or
 * SMAPB_JPEG_UNSUPPORTED once the data is decoded.  Each phase is one launch for the whole batch.  The workspace is owned
 * by the handle and grows on demand; the call synchronises `stream` and returns once status_host is known, so it cannot be
 * captured into a CUDA graph. */
int smapb_decode_jpeg(smapb_handle* h, int n, const uint8_t* const* jpeg_host, const int64_t* nbytes, uint8_t* const* bgr_dev,
                      int* status_host, void* stream);
/* Flags of the _ex forms; 0 = exactly smapb_jpeg_info / smapb_decode_jpeg.
 * SMAPB_JPEG_SCANS also accepts sequential files (SOF0/SOF1) with several scans (every component in exactly one) and
 * progressive Huffman files (SOF2) whose progression libjpeg accepts without a warning and whose coefficients 1..9 are
 * fully refined in every component (otherwise libjpeg-turbo smooths the output, and the file is left to cv2), with at
 * most 64 scans and no DQT redefining a table a scan already used.  One call decodes a mixed batch (single-scan,
 * multi-scan and refused files); the status codes, the shape rule and the synchronisation are those of the plain forms.
 * AC refinement scans decode sequentially within a restart segment (a block's bits depend on its coefficients' history),
 * one warp per segment against per-block history masks; the segments, and the images of a batch, run side by side. */
#define SMAPB_JPEG_SCANS 1
/* SMAPB_JPEG_COLOUR (alone or with SMAPB_JPEG_SCANS) also accepts the frames libjpeg reads that the plain forms leave to
 * cv2 for their colour space or sampling: 4 components (CMYK, or YCCK when an Adobe APP14 says transform 2; other Adobe
 * transforms are left to cv2), 3 components libjpeg treats as RGB (an Adobe transform of 0 without JFIF, or ids 'R','G','B'
 * without either marker), and every sampling with factors H, V in 1..4 whose ratios to the frame's largest factors are
 * integral (4:1:1, 4:1:0, factors of 3, chroma finer than luma, Pillow's CMYK with the factors on C) and at most 10 blocks
 * per MCU.  Each component is upsampled as libjpeg-turbo 3.x does it (fancy h2v1 / h1v2 / h2v2 where a factor is halved,
 * replication for other ratios); RGB is reordered to BGR, and CMYK (YCCK first converted to CMYK with the YCbCr tables)
 * goes through cv2's CMYK -> BGR, out = K - ((255 - ink) * K >> 8).  Still left to cv2: fractional sampling ratios, frames
 * over 10 blocks per MCU, 2-component frames, arithmetic coding, 12-bit and lossless files. */
#define SMAPB_JPEG_COLOUR 2
int smapb_jpeg_info_ex(const uint8_t* data, int64_t nbytes, int flags, int* h, int* w, int* orientation, int* status);
int smapb_decode_jpeg_ex(smapb_handle* h, int n, const uint8_t* const* jpeg_host, const int64_t* nbytes, uint8_t* const* bgr_dev,
                         int flags, int* status_host, void* stream);

/* ---- PNG decoding (the step in front of pre-processing) -------------------------------------------------------------- */
/* Replaces: cv2.imread(path, IMREAD_COLOR) (dataset/custom_dataset.py:27) for the PNGs it can decode, byte for byte: every
 * legal bit depth / colour type pair (grey 1/2/4/8/16, RGB 8/16, palette 1/2/4/8, grey+alpha and RGBA 8/16), interlace 0
 * and Adam7, any zlib stream (stored, fixed and dynamic blocks, any level, strategy, window and flush) in IDATs of any
 * size, eXIf orientation 1..8 applied as cv2 applies it, up to SMAPB_JPEG_MAX_PIXELS.  As cv2 does, it keeps the high byte
 * of 16-bit samples, drops alpha without compositing, replicates grey, scales 1/2/4-bit grey to 8 bits, reads a palette
 * index past PLTE's entries as black and ignores tRNS, gAMA, sBIT, bKGD and colour management.  Everything else (APNG, an
 * unknown critical chunk, a PLTE in a grey image, a CRC error in any chunk, a bad zlib header, preset dictionaries, a
 * stream that does not inflate to exactly the scanlines' bytes, data after its Adler-32, non-PNG data) gets a status
 * != SMAPB_JPEG_OK and is meant for cv2.imread; every file cv2 refuses is among them.  Two kinds of valid stream that
 * cv2 reads are among them too: more DEFLATE blocks than (zlib stream bytes) / 8 + 64, and a match reaching past the
 * window the zlib header declares.  The statuses are SMAPB_JPEG_*. */
/* Host only (no GPU work): chunk walk of one file.  *status = SMAPB_JPEG_*; when it is SMAPB_JPEG_OK, *h x *w is the shape
 * cv2.imread returns (after the EXIF orientation) and *orientation the EXIF value (1 without one); zeros otherwise.
 * Returns 0, or -1 for a NULL status. */
int smapb_png_info(const uint8_t* data, int64_t nbytes, int* h, int* w, int* orientation, int* status);
/* Decodes n files (host memory) into bgr_dev[i]: uint8 [h, w, 3] BGR as smapb_png_info reports the shape, which
 * smapb_preprocess consumes.  bgr_dev[i] may be NULL only for files smapb_png_info does not accept.  status_host[i]
 * (SMAPB_JPEG_*) says whether bgr_dev[i] holds the image; the header status can turn into SMAPB_JPEG_CORRUPT (an IDAT CRC,
 * the Adler-32, a code or distance zlib refuses, too little data) or SMAPB_JPEG_UNSUPPORTED once the data is inflated.
 * The zlib streams are inflated block-parallel: a block finder lists candidate dynamic-block headers, which are decoded
 * side by side, and a walk from each stream's first block keeps the real ones and decodes the rest itself.  Each phase is
 * one launch for the whole batch.  The workspace is owned by the handle and grows on demand; the call synchronises
 * `stream` and returns once status_host is known, so it cannot be captured into a CUDA graph. */
int smapb_decode_png(smapb_handle* h, int n, const uint8_t* const* png_host, const int64_t* nbytes, uint8_t* const* bgr_dev,
                     int* status_host, void* stream);

/* ---- backbone -------------------------------------------------------------------------------- */
/* Replaces: SMAP.forward inference branch (model/smap.py:403-419).
 * imgs_nchw_dev: fp32 [B,3,in_h,in_w] (normalised BGR).  Outputs fp32 NCHW:
 * hm2d [B,43,h,w], detd [B,14,h,w], rootd [B,1,h,w] with h=in_h/4, w=in_w/4. */
int smapb_backbone_forward(smapb_handle* h, const float* imgs_nchw_dev, int B, float* hm2d_dev, float* detd_dev,
                           float* rootd_dev, void* stream);
/* Flip-TTA merge (exps/stage3_root2/test.py:55-70) and the per-image rescale hms[:15]/=255,
 * hms[15:]/=127 (exps/stage3_root2/test.py:111-112), in place on hm2d [B,43,h,w].
 * hm2d_flip_dev may be NULL (no TTA).  do_scale != 0 applies the division. */
int smapb_merge_scale(smapb_handle* h, float* hm2d_dev, const float* hm2d_flip_dev, int B, int do_scale,
                      void* stream);

/* ---- association ----------------------------------------------------------------------------- */
/* Replaces: dapalib.extract (extensions/association.cpp:34-120): nmsGpu + connectBodyPartsGpu.
 * hms_dev: fp32 [B,43,h,w] already divided by 255/127.
 * peaks_dev: fp32 [B,15,128,3]  slot 0 = (count,0,0), slots 1..count = (x,y,score) in raster order,
 *            remaining slots zero (the reference leaves them uninitialised).
 * pair_scores_dev: fp32 [B,14,127,127], -1 outside nA x nB exactly as pafScoreKernel writes. */
int smapb_assoc_extract(smapb_handle* h, const float* hms_dev, int B, float* peaks_dev, float* pair_scores_dev,
                        void* stream);
/* Replaces: dapalib.connect / findConnectedJoints (extensions/association.cpp:123-233).
 * rdepth_dev: fp32 [B,h,w].  bodies_dev: fp32 [B,127,15,4] = (x,y,0,score) in heat-map pixels, rows in
 * ascending root depth, rows >= counts[b] zero.  counts_dev: int32 [B]. */
int smapb_assoc_connect(smapb_handle* h, const float* hms_dev, const float* rdepth_dev, int B, int root_idx,
                        int dist_flag, float* bodies_dev, int* counts_dev, void* stream);

/* ---- 3D lift ---------------------------------------------------------------------------------- */
/* Replaces: x4 stride + nearest upsample + register_pred(no GT) + generate_relZ + gen_3d_pose
 * (exps/stage3_root2/test.py:117-134, test_util.py:18-99, lib/utils/post_3d.py:4-27).
 * scales_dev: float64 [B,9] (SMAPB_SCALE_LEN).  Outputs (fixed stride, tails zeroed):
 * pred2d fp32 [B,127,15,4] (x,y in net-input pixels, root-relative z, score),
 * pred3d fp64 [B,127,15,4] (X,Y,Z,score), root_depth fp64 [B,127], counts_out int32 [B]. */
int smapb_lift3d(smapb_handle* h, const float* bodies_dev, const int* counts_dev, const float* detd_dev,
                 const float* rootd_dev, const double* scales_dev, int B, float* pred2d_dev, double* pred3d_dev,
                 double* root_depth_dev, int* counts_out_dev, void* stream);

/* The same with ground truth: the matching branch of register_pred (exps/stage3_root2/test_util.py:21-39) used by the
 * reference's `generate_result` / `generate_train` test modes (exps/stage3_root2/test.py:73-95,129).  gt_roots_dev: float64
 * [B,gmax,2] = gt_bodys[:, ROOT_IDX, :2] (network-input pixels) of the persons test.py:80-82 keeps, gt_counts_dev int32 [B].
 * Predictions are matched to GT persons greedily by ascending root distance below 30 px (ties in row-major order); output
 * row g belongs to GT person g (all-zero when unmatched), counts_out[b] = gt_counts[b] (0 when the frame has no
 * prediction or no GT person - the reference skips it).  In this branch the body rows are float64 (np.zeros(..., np.float),
 * test_util.py:35), so pred2d is float64 [B,127,15,4] as well; scales_dev carries the GT intrinsics (test.py:86-95). */
int smapb_lift3d_gt(smapb_handle* h, const float* bodies_dev, const int* counts_dev, const float* detd_dev,
                    const float* rootd_dev, const double* scales_dev, const double* gt_roots_dev, const int* gt_counts_dev,
                    int gmax, int B, double* pred2d_dev, double* pred3d_dev, double* root_depth_dev, int* counts_out_dev,
                    void* stream);

/* ---- whole path -------------------------------------------------------------------------------- */
/* Byte layout of one per-image skeleton record (the all-gather payload, SURVEY.md 8(e)). */
typedef struct smapb_record {
    double pred3d[SMAPB_MAXP][SMAPB_NJ][4];
    double root_depth[SMAPB_MAXP];
    float pred2d[SMAPB_MAXP][SMAPB_NJ][4];
    int32_t count;
    int32_t pad_;
} smapb_record;

/* Replaces: the per-batch body of generate_3d_point_pairs (exps/stage3_root2/test.py:48-134) with
 * device-resident input: forward (+ flipped forward when do_flip) -> merge/scale -> connect -> lift.
 * records_dev: smapb_record[B]. */
int smapb_infer_device(smapb_handle* h, const float* imgs_nchw_dev, const double* scales_dev, int B, int do_flip,
                       smapb_record* records_dev, void* stream);
/* Same with HOST buffers (pinned or pageable): H2D of imgs/scales, infer, D2H of records, then
 * synchronises `stream`.  This is the call bench.py times as `e2e`. */
int smapb_infer_host(smapb_handle* h, const float* imgs_nchw_host, const double* scales_host, int B, int do_flip,
                     smapb_record* records_host, void* stream);

/* Pipelined form of smapb_infer_host for streams of batches: two slots (0/1).  smapb_submit_host enqueues H2D (on a copy
 * stream), the whole path and the D2H of the records for one batch and returns immediately; smapb_wait blocks until that
 * slot's records are in `records_host`.  Submitting to slot s while slot 1-s computes overlaps the next batch's H2D with
 * the current batch's compute.  Host buffers must stay valid (and should be pinned) until smapb_wait returns. */
int smapb_submit_host(smapb_handle* h, int slot, const float* imgs_nchw_host, const double* scales_host, int B, int do_flip,
                      smapb_record* records_host);
int smapb_wait(smapb_handle* h, int slot);

/* ---- multi-GPU: frames are sharded over ranks, ONE exchange step per batch --------------------------------------- */
/* The reference's inference path is single-GPU (exps/stage3_root2/test.py:198 calls get_test_loader with num_gpu=1);
 * its data loader's rank split (lib/utils/dataloader.py:80-85: contiguous blocks of frames per rank) is the sharding
 * rule used here, and the only exchange is one ncclAllGather of the fixed-stride smapb_record[B] per batch
 * (SURVEY.md 8(e)).  NCCL is bound at run time (dlopen of libnccl.so.2 - inside a PyTorch process that is the instance
 * torch loaded), so the library has no link-time dependency on it and a communicator may come from either side:
 *   smapb_comm_unique_id + smapb_comm_create : the handle creates (and owns) its communicator; rank 0 makes the
 *       128-byte ncclUniqueId, the host side distributes it (any transport), every rank calls smapb_comm_create.
 *   smapb_comm_attach : borrow an existing ncclComm_t (e.g. torch.distributed's ProcessGroupNCCL._comm_ptr()).
 * One communicator per handle: two handles of a rank keep two batches in flight without ordering constraints
 * between their collectives. */
int smapb_comm_unique_id(void* id128 /* out: 128 bytes */);
int smapb_comm_create(smapb_handle* h, const void* id128, int rank, int world);
int smapb_comm_attach(smapb_handle* h, void* nccl_comm /* ncclComm_t, caller-owned */, int rank, int world);
/* The exchange step by itself: all-gather B records per rank into all_records_dev[world * B] (rank order), on `stream`.
 * nccl_comm NULL = the handle's communicator. */
int smapb_allgather_records(smapb_handle* h, void* nccl_comm, const smapb_record* records_dev, smapb_record* all_records_dev,
                            int B, void* stream);
/* smapb_infer_device / smapb_submit_host followed by the all-gather on the SAME stream, inside the same CUDA graph
 * (set SMAPB_NCCL_EAGER=1 to keep the collective outside the graph, still stream-ordered): all_records receives
 * world * B records in rank order - the frames of the global batch in their original order.  The host variant gathers
 * on the device (NVLink) and then performs a single D2H of the gathered records. */
int smapb_infer_device_gather(smapb_handle* h, const float* imgs_nchw_dev, const double* scales_dev, int B, int do_flip,
                              smapb_record* all_records_dev, void* stream);
int smapb_submit_host_gather(smapb_handle* h, int slot, const float* imgs_nchw_host, const double* scales_host, int B,
                             int do_flip, smapb_record* all_records_host);
/* Decoupled form for streams of batches (what bench.py times at N > 1): the whole path is enqueued on `stream`, the all-gather
 * on the handle's own gather stream behind an event - `stream` is ordered after the COMPUTE only, so a rank's compute stream
 * never waits for its peers (the stream-ordered form above locks the ranks into step with each other - not in the
 * 14 us collective but in the lock-step it imposes on the ranks' two batches in flight; this form costs nothing).
 * all_records_dev is valid once smapb_gather_sync(h, s) has made a stream s wait for the outstanding exchanges.  The records
 * are double-buffered inside the handle: a call waits at most for the exchange issued two calls earlier.
 * smapb_submit_host_gather uses the same side stream (its smapb_wait covers the exchange and the D2H). */
int smapb_infer_device_gather_async(smapb_handle* h, const float* imgs_nchw_dev, const double* scales_dev, int B, int do_flip,
                                    smapb_record* all_records_dev, void* stream);
int smapb_gather_sync(smapb_handle* h, void* stream);

/* ---- RefineNet post-processing (optional; the reference enables it with `-rp`, exps/stage3_root2/test.sh) ------- */
/* Replaces: refine_model.load_state_dict(torch.load(path)) (exps/stage3_root2/test.py:213-214) for model/refinenet.py:
 * keys "block.layer{1..4}.0.{weight,bias}" (Linear), "block.layer{1..4}.1.{weight,bias,running_mean,running_var}"
 * (BatchNorm1d), "block.layer5.{weight,bias}"; num_batches_tracked is accepted and ignored. */
int smapb_refine_load_weight(smapb_handle* h, const char* key, const float* host, const int64_t* shape, int ndim);
/* BN folding (eval mode, eps 1e-5) + transposition; must follow the last smapb_refine_load_weight. */
int smapb_refine_finalize(smapb_handle* h);
/* Replaces: refine_model(inp) (model/refinenet.py:19-26, eval): in fp32 [n,75] -> out fp32 [n,45], device pointers. */
int smapb_refine_mlp(smapb_handle* h, const float* in_dev, int n, float* out_dev, void* stream);
/* Replaces: lift_and_refine_3d_pose (exps/stage3_root2/test_util.py:102-131) for a batch of images, device-resident:
 * pred2d fp32 [B,127,15,4], pred3d fp64 [B,127,15,4], counts int32 [B] (the outputs of smapb_lift3d) ->
 * refined fp64 [B,127,15,4] = (X,Y,Z,score), rows >= counts[b] untouched.  refined may alias pred3d. */
int smapb_refine3d(smapb_handle* h, const float* pred2d_dev, const double* pred3d_dev, const int* counts_dev, int B,
                   int root_idx, double* refined_dev, void* stream);
/* enable != 0: smapb_infer_device / _host / smapb_submit_host run the refinement after the lift and store the refined
 * poses in smapb_record.pred3d, as generate_3d_point_pairs saves new_pred_bodys_3d (exps/stage3_root2/test.py:136-145). */
int smapb_set_refine(smapb_handle* h, int enable);

/* ---- result serialisation (host only, no GPU work) ------------------------------------------------------- */
/* Replaces: result = {'model_pattern': cfg.DATASET.NAME, '3d_pairs': []} ... save_result(...) per image ...
 * json.dump(result, f) (exps/stage3_root2/test.py:32-34,145,147-152; exps/stage3_root2/test_util.py:146-158) for the
 * run_inference mode (no ground truth).  The file is byte-identical to what Python's json.dump writes for the same
 * numbers (float repr, ", " / ": " separators, ensure_ascii escaping, key order of save_result). */
typedef struct smapb_json_writer smapb_json_writer;
int smapb_json_open(smapb_json_writer** out, const char* path, const char* model_pattern);
/* Appends one entry per record with count > 0 (images without persons are skipped, test.py:130-131).
 * records_host: smapb_record[B] in host memory; image_paths: B UTF-8 strings. */
int smapb_json_append(smapb_json_writer* w, const smapb_record* records_host, int B, const char* const* image_paths);
/* Writes the closing brackets, closes the file and frees the writer. */
int smapb_json_close(smapb_json_writer* w);

/* ---- introspection ----------------------------------------------------------------------------- */
/* number of kernels launched by this handle since creation */
int64_t smapb_launch_count(const smapb_handle* h);
/* SMAPB_PREC_FP16: number of activation elements this handle's kernels clamped to +-65504 since creation (or the last
 * reset != 0, which zeroes the counter after reading it); 0 in the bf16 precisions.  Every forward (eager, graph replay,
 * each half of a flip pass, a profiled run) and each smapb_conv_test call adds its clamps once; the autotuner's trial
 * launches at plan build and smapb_conv_test's timed re-runs add nothing.  Synchronises the device.  Any nonzero
 * count means some layer produced values fp16 cannot hold and those outputs are not the model's: run such inputs (or
 * weights) with SMAPB_PREC_BF16X3, or SMAPB_PREC_BF16 when speed matters more than the last digits.  < 0: error. */
int64_t smapb_saturation_count(smapb_handle* h, int reset);
/* Per-op device timing with CUDA events on the launching stream (bench.py roofline leg).  After
 * smapb_profile_begin every kernel launched through this handle is bracketed by events; smapb_profile_end
 * synchronises the device, sums milliseconds and launch counts per kind
 * (0 conv_tc, 1 stem+maxpool, 2 other backbone elementwise, 3 association, 4 lift, 5 unused) into the two
 * 6-element arrays and, if csv_path is not NULL, writes one line per launch. */
int smapb_profile_begin(smapb_handle* h);
int smapb_profile_end(smapb_handle* h, double* ms_by_kind, int* launches_by_kind, const char* csv_path);
/* Tile shapes of the tensor-core convolutions (process-wide): one line per layer geometry, "key<TAB>BLOCK_N<TAB>variant"
 * (BLOCK_N: 32, 64 or 128 output channels per 128-row tile; variant: 1 = one CTA per tile, the only one the sm_90a kernel has;
 * entries it cannot run are stored but measured again).  Whatever shape computes a layer, the result bits are the same.
 * Geometries found in the table with a shape the kernel has use its entry; others are autotuned once per process (SMAPB_NO_AUTOTUNE=1: cost model)
 * and added to it.  Loading the same table in every process makes tile selection - and with it every result bit -
 * independent of the handle, the process and the rank.  smapb_get_tile_table returns the bytes needed (incl. the
 * terminating 0) and fills buf up to cap. */
int smapb_set_tile_table(const char* text);
int smapb_get_tile_table(char* buf, int cap);
/* conv plan: number of tensor-core conv launches per forward and their algorithmic FLOPs (2*MACs, 1x) */
int smapb_plan_info(const smapb_handle* h, int B, int* n_conv_launches, double* conv_flops);
/* Run one standalone convolution through the tensor-core path (test/bench hook), with every epilogue form the plan uses.
 * x: fp32 NHWC [B,H,W,Cin]; w: fp32 [Cout,Cin+Cin2,k,k]; bias fp32 [Cout]; padding k/2, Ho = (H + 2 (k/2) - k) / stride + 1
 * (likewise Wo).  Optional inputs (NULL = absent), converted to the precision's planes as the plan's activations are:
 *   res        fp32 NHWC [B,Ho,Wo,Cout] added before the ReLU;
 *   post1/2    fp32 NHWC [B,Ho,Wo,Cout] added after the ReLU, in that order (post2 needs post1);
 *   in2        fp32 NHWC [B,H2,W2,Cin2], the K-concatenated second input of a fused pair: its 1x1 conv with stride stride2
 *              (weight columns Cin .. Cin+Cin2-1) joins the same accumulation; needs k = 1, stride = 1, Cin2 % 64 == 0 and
 *              (H2-1)/stride2 + 1 == Ho, (W2-1)/stride2 + 1 == Wo.  Cin2 = 0 without it;
 *   up         fp32 NHWC [B,Ho/2,Wo/2,Cout], up-sampled x2 (bilinear, align_corners=True) and added before the ReLU; not
 *              with res or post1.
 * res, post1, post2 and up need Cout % 32 == 0.  out_f32 != 0: the conv stores fp32, as the plan's head convs do, instead
 * of the precision's activation planes.  y: fp32 NHWC [B,Ho,Wo,Cout], the stored output's value.  launch (optional,
 * int[4]) receives what the result launch ran: BLOCK_N, the patch width tw (128 in the flat mode), 1 for the flat mode
 * (1x1 stride-1 convs see N*Ho*Wo pixels as one row) or 0 for patch tiles, and the epilogue-input ring (0 none,
 * 1 residual / skips, 2 up-residual).  All tensors are device pointers.  A combination the plan's conv set-up refuses is
 * refused here with its error message (smapb_last_error). */
int smapb_conv_test(smapb_handle* h, const float* x_dev, const float* w_dev, const float* bias_dev,
                    const float* res_dev, const float* post1_dev, const float* post2_dev, const float* in2_dev,
                    const float* up_dev, int B, int H, int W, int Cin, int Cout, int k, int stride, int H2, int W2,
                    int Cin2, int stride2, int relu, int out_f32, int precision, float* y_dev, int* launch, float* ms_out,
                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SMAP_B200_H */
