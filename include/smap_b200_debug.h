/*
 * smap_b200 - debug / bisection entry points of libsmap_b200.so.  NOT part of the drop-in boundary (include/smap_b200.h);
 * used by tools/debug_*.py to localise numerical differences op by op.  They synchronise the device.
 */
#ifndef SMAP_B200_DEBUG_H
#define SMAP_B200_DEBUG_H

#include "smap_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* 64-bit position-weighted checksums of the output tensor of every op of the batch-B plan, as left by the last forward.
 * sums[max_ops]; desc (optional): max_ops strings of desc_stride bytes (512 is enough) describing each op.  Returns the number
 * of ops.  Op i here is dump index i of smapb_debug_dump.  A description is space-separated key=value fields:
 *   name=<unit name>  kind=conv | conv_f32 | stem_tc | stem | s2d | maxpool
 *     conv: tensor-core conv with split-bf16 output; conv_f32: fp32 NHWC output (heads, *.tapexp); stem_tc: the 7x7/s2
 *     stem as a 4x1-tap conv over the s2d view; stem: the CUDA-core stem; s2d: space-to-depth of the image
 *   inputs by role, as dump indices, absent roles left out: in= res= p1= p2= in2= up= (convs), a= (maxpool);
 *     in=x is the network input image
 *   convs:  tw= (patch width; 128 on the flat path) k=<kh>x<kw> s= pad=<y>x<x> cin= cin2= s2=
 *           cout= (padded) out=NxHxWxC bn= relu= hasres= post= upmode= tiles= nterms=
 *   others: out=NxHxWxC nterms= */
int smapb_debug_checksums(smapb_handle* h, int B, unsigned long long* sums, int max_ops, char* desc, int desc_stride);
/* Raw copy (both bf16 planes, or fp32 for head outputs) of op `idx`'s output into host or device memory (the copy direction
 * is inferred from the pointer); returns the bytes copied. */
long long smapb_debug_dump(smapb_handle* h, int B, int idx, void* host, long long max_bytes, int which);

/* Host-only: the resampling plan smapb_preprocess uses for a src_w x src_h image (no GPU work).  dims6 = {dst_w, dst_h,
 * pad_left, pad_top, mode (0 fixed-point bilinear, 1 exact 1/2 scale = 2x2 rounded mean, 2 copy), 0}; the tables (may be
 * NULL) must hold dst_w, 2*dst_w, 2*dst_h and 2*dst_h entries (dst <= net size).  Returns -1 for a geometry
 * smapb_preprocess refuses. */
int smapb_debug_resize_plan(int src_w, int src_h, int net_w, int net_h, int* dims6, double* scale, int* xofs, short* xcoef,
                            int* yofs, short* ycoef);

/* Inflate counters of the handle's last smapb_decode_png call: counts4 = {candidates the block finder listed, false
 * positives (candidates no chained block starts at), chained blocks confirmed through the finder, chained blocks the
 * serial walk handled itself (stored, fixed-Huffman, and dynamic blocks the finder missed or could not confirm)}.
 * Zeros before the first call. */
int smapb_png_inflate_stats(const smapb_handle* h, int64_t* counts4);

/* Environment switches read when a handle / plan is built (never on the per-call path):
 *   SMAPB_DEBUG_STOP=n        run only the first n ops of the plan
 *   SMAPB_DEBUG_SYNC=1        synchronise the stream after every launch
 *   SMAPB_FORCE_TILE=bn       force a tile width (32, 64, 128) wherever it is valid, except where the tile table or the
 *                             autotuner picks one;  SMAPB_NO_AUTOTUNE=1  cost model only
 *   SMAPB_NO_GRAPH=1          no CUDA graph replay
 *   SMAPB_STEM=cuda           CUDA-core stem
 *   SMAPB_ROLES=1             per-role wait-cycle counters in smapb_conv_test
 *   SMAPB_ROLES_PLAN=file.csv the same counters for every conv launch of a profiled (smapb_profile_begin/end) run, i.e. inside the
 *                             real step (tools/roles_plan.py)
 *   SMAPB_TIMELINE=1          clock64 time line of CTA 0 of one launch in smapb_conv_test (set-up, first operands, last main loop end,
 *                             epilogue done, exit)
 *   SMAPB_JPEG_SUB_BITS=n     subsequence length (bits, a multiple of 32) of the Huffman passes of every JPEG decode
 *                             (smapb_decode_jpeg[_ex]); default 512; short ones make blocks and EOB runs cross subsequence
 *                             boundaries in tests
 *   SMAPB_LIB=path (Python)   load another build of the library (A/B runs: tools/ab_hash.py) */

#ifdef __cplusplus
}
#endif
#endif /* SMAP_B200_DEBUG_H */
