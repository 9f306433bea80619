// Implicit-GEMM convolution on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
//   y[n, oy, ox, co] = epilogue( sum_{ky,kx,ci} x[n, oy*s+ky-p, ox*s+kx-p, ci] * w[co, ci, ky, kx] )
//
// GEMM view: M = output pixels (a th x tw spatial patch = 128 rows per tile), N = Cout, K = taps * Cin.
// One k-block = one filter tap x 64 input channels.  Operands are K-major 2-byte (bf16 or fp16) tiles of 128-byte rows in
// SWIZZLE_128B shared-memory layout, written by TMA:
//   A: 5-D tensor map (C, W, H, N, term) over the NHWC activation planes; the tap shift is a coordinate
//      offset, zero padding is TMA out-of-bounds fill, conv stride is the map's elementStrides.
//   B: 4-D tensor map (Cin, Cout, tap, term) over the repacked (BN-folded) weights.
// Precision: "bf16x3" - every fp32 value v is carried as two bf16 planes (hi = bf16(v), lo = bf16(v - hi));
// a product a*b is issued as 3 MMAs  a_hi*b_hi + a_lo*b_hi + a_hi*b_lo  into the same fp32 accumulator
// (dropped terms are O(2^-16) relative) - fp32-faithful results at 3x the bf16 MMA count.  NTERMS = 1 is the
// plain bf16 fast mode.  With E = ElemF16 (NTERMS = 1) operands and stored activations are fp16 (same bytes, same MMA rate,
// 4x finer rounding than bf16); the epilogue clamps every stored value to +-65504 and counts the clamped elements in p.sat.
//
// Roles (384 threads, persistent CTA, static tile schedule; every role branch is warpgroup-uniform, registers are
// rebalanced per role with setmaxnreg):
//   warpgroup 0 (40 registers) : warp 0 = operand TMA producer (one lane), warp 1 = epilogue-input TMA producer (one lane)
//   warpgroups 1-2 (232 registers) : ping-pong consumers.  The CTA's tiles alternate between them: warpgroup g runs tiles
//                g, g + 2, ... of the CTA's list, each a whole 128-row tile issued as two m64nBLOCK_Nk16 row halves into
//                registers, then the epilogue from those registers in 32-column chunks: (+bias +residual, ReLU, +skips,
//                hi/lo split) -> the warpgroup's swizzled staging slot -> one TMA store per chunk and plane.
//                Main loops are handed from one warpgroup to the other in tile order (a named-barrier token), so one
//                warpgroup's epilogue runs while the other issues the next tile's wgmma.
// Pipelines: operand full/empty ring (TMA <-> wgmma, consumed tile by tile in the CTA's tile order), epilogue-input
// full/empty ring (TMA <-> epilogue, one FIFO in the same tile order), bulk-async store groups (per warpgroup leader).
// Taps of a k x k filter are visited kx-major and every tile width issues the same MMAs per output element in the same
// order, i.e. all tile shapes produce the same bits.
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace smapb {

struct alignas(64) ConvParams {
    CUtensorMap tmA;  // activations (loads)
    CUtensorMap tmA2; // second activation tensor of a K-concatenated 1x1 pair (conv3 + downsample), or unused
    CUtensorMap tmB;  // weights (loads)
    CUtensorMap tmO;  // output planes (stores, 32-channel boxes, SWIZZLE_64B)
    CUtensorMap tmR[3];  // epilogue input planes (loads, same geometry as tmO): [residual][post1][post2] as present
    // geometry
    int Hout, Wout, Nimg;
    int tw_log2, th;  // tile: tw = 1 << tw_log2, tw * th == 128
    int tiles_x, tiles_y;
    int Cout;  // channel stride of the output / residual tensors (elements)
    int kh, kw, stride, pad_y, pad_x;  // filter taps (kh x kw), spatial stride, zero padding
    int kchunks;  // Cin / 64
    int kchunks2, stride2;  // K-concatenated second 1x1 input: Cin2 / 64 (0 = none) and its spatial stride
    int n_tiles;  // Cout_pad / BLOCK_N
    int total_tiles;
    // epilogue
    const float* bias;           // [Cout_pad] folded bias
    int has_res;  // tmR[0] is a residual added before the ReLU (model/smap.py:74-75)
    int n_post;   // number of tensors added after the ReLU (x_k = layer_k + skip1 + skip2, model/smap.py:143)
    __nv_bfloat16* out;  // bf16 hi/lo planes NHWC, or null
    float* out_f32;      // fp32 NHWC (heads), or null
    long long plane_stride;  // elements between the hi and lo planes (= N*H*W*Cout)
    int relu;
    int reverse;    // walk the tile list back to front (the consumer of a tensor starts with the rows its producer wrote
                    // last, which are the ones still resident in L2)
    // fused bilinear residual (Upsample_unit, model/smap.py:211-217): tmR[0] is a low-resolution tensor [N,Hi,Wi,C];
    // the ring carries the (ph x pw)-pixel patch under each output tile and the epilogue interpolates
    // (align_corners=True) before the ReLU.  up_mode = 0: plain residual.
    int up_mode, up_Hi, up_Wi, up_pw, up_ph;
    long long* dbg;  // optional: per-role cycle counters, layout ConvDbg below (tools/roles_plan.py), null in production
    long long* dbg_tl;  // optional: clock64 time line of CTA 0 (SMAPB_TIMELINE, smapb_conv_test only), null in production
    unsigned long long* sat;  // fp16 kernels: count of stored elements clamped to +-65504 (the handle's saturation counter)
};

// ---- TMA / wgmma PTX wrappers -------------------------------------------------------------------
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, "
        "%7}], [%2];" ::"r"(dst),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, "
        "%6}], [%2];" ::"r"(dst),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3,
                                             int c4) {
    asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(map),
                 "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// Named barriers (0 is __syncthreads): 1 + g = epilogue of consumer warpgroup g (128 threads).  Turns (2 x 128 threads,
// synced by warpgroup g, arrived at by the other consumer warpgroup when it is done with its previous tile):
// 3 + g = main-loop turn of g, 5 + g = epilogue-input ring turn of g
enum { TURN_MAIN = 3, TURN_RING = 5 };
__device__ __forceinline__ void epi_bar_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }
__device__ __forceinline__ void turn_wait(int turn, int wg) { asm volatile("bar.sync %0, 256;" ::"r"(turn + wg) : "memory"); }
__device__ __forceinline__ void turn_pass(int turn, int wg) { asm volatile("bar.arrive %0, 256;" ::"r"(turn + wg) : "memory"); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
// Per-role cycle counters (p.dbg != null), summed over CTAs.  Consumer warpgroup g uses CONS + CONS_N g + {...}.
struct ConvDbg {
    enum {
        PRODUCER_WAIT_EMPTY = 0,  // operand producer waiting for a free stage
        TOTAL = 1,                // CTA lifetime from set-up to exit
        CTAS = 2,                 // number of CTAs that added to the counters
        CONS = 3,
        WAIT_FULL = 0,   // operands not yet landed
        WAIT_ORDER = 1,  // waiting for the main-loop turn (the other warpgroup still issuing its tile)
        EPILOGUE = 2,    // time in epilogues
        WAIT_RING = 3,   // epilogue inputs not yet landed
        WAIT_STAGE = 4,  // own staging slot still being read by the previous TMA store
        CONS_N = 5,
        COUNT = CONS + 2 * CONS_N
    };
};
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
    uint32_t r;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(addr));
    return r;
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// byte offset of 16-byte chunk j (0..3) of row r in a [rows x 64 B] SWIZZLE_64B box
__device__ __forceinline__ uint32_t sw64_off(int r, int j) { return (uint32_t)(r * 64 + ((j ^ ((r >> 1) & 3)) << 4)); }

// ATen bilinear, align_corners=True: src = dst * (in-1)/(out-1) in fp32; i0 = (int)src
__device__ __forceinline__ float up_scale(int in, int out) { return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f; }
__device__ __forceinline__ int up_src_index(int dst, int in, int out) { return (int)(up_scale(in, out) * (float)dst); }

// the fp32 values (low half, high half) a hi/lo pair of bf16x2 words carries: hi + lo, exact widening, one rounding
__device__ __forceinline__ float2 planes_to_f2(uint32_t h, uint32_t l) {
    return make_float2(bf16lo_to_f(h) + bf16lo_to_f(l), bf16hi_to_f(h) + bf16hi_to_f(l));
}

// wgmma shared-memory operand descriptor: K-major, SWIZZLE_128B, rows of 128 B, 8-row groups 1024 B apart (SBO);
// LBO is unused for swizzled K-major operands.  A k-step of 16 bf16 (32 B) inside the swizzle atom adds 2 to the address.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;  // SWIZZLE_128B
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// D[64 x N] (+)= A[64 x 16] * B[16 x N]^T, fp32 accumulators in the wgmma fragment layout: thread t of the warpgroup holds
// rows 16 (t / 32) + (t % 32) / 4 + {0, 8} and columns 8 j + 2 (t % 4) + {0, 1} as d[4 j + 2 {0, 1} + {0, 1}]
template <class E>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
#define SMAPB_WGMMA(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, " \
        "%13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, " \
        "%36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, " \
        "%59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), \
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), \
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), \
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), \
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), \
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), \
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), \
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
        : "l"(adesc), "l"(bdesc), "r"(accumulate))
    if constexpr (E::F16) SMAPB_WGMMA("f16");
    else SMAPB_WGMMA("bf16");
#undef SMAPB_WGMMA
}
template <class E>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
#define SMAPB_WGMMA(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, " \
        "%13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, " \
        "1, 0, 0;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), \
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), \
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), \
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
        : "l"(adesc), "l"(bdesc), "r"(accumulate))
    if constexpr (E::F16) SMAPB_WGMMA("f16");
    else SMAPB_WGMMA("bf16");
#undef SMAPB_WGMMA
}
template <class E>
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
#define SMAPB_WGMMA(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, " \
        "%13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), \
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
        : "l"(adesc), "l"(bdesc), "r"(accumulate))
    if constexpr (E::F16) SMAPB_WGMMA("f16");
    else SMAPB_WGMMA("bf16");
#undef SMAPB_WGMMA
}
template <int BLOCK_N, class E>
__device__ __forceinline__ void wgmma_tile(float (&d)[BLOCK_N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    if constexpr (BLOCK_N == 128) wgmma_m64n128<E>(d, adesc, bdesc, accumulate);
    else if constexpr (BLOCK_N == 64) wgmma_m64n64<E>(d, adesc, bdesc, accumulate);
    else wgmma_m64n32<E>(d, adesc, bdesc, accumulate);
}

// mbar_wait that also returns the cycles spent waiting (role-level profiling; only used when p.dbg != null)
__device__ __forceinline__ long long mbar_wait_timed(uint64_t* bar, uint32_t parity, bool timed) {
    if (!timed) {
        mbar_wait(bar, parity);
        return 0;
    }
    const long long t0 = clock64();
    mbar_wait(bar, parity);
    return clock64() - t0;
}

// RING: 0 = no epilogue inputs, 1 = residual / skip tensors through the ring, 2 = fused bilinear residual (up_mode)
template <int BLOCK_N, int NTERMS, int RING>
struct ConvCfg {
    static constexpr int TA = (NTERMS == 3) ? 2 : 1;  // operand planes held per stage
    static constexpr int A_BYTES = 128 * 128;         // rows x 64 bf16
    static constexpr int B_BYTES = BLOCK_N * 128;
    static constexpr int STAGE_BYTES = TA * (A_BYTES + B_BYTES);
    static constexpr int CHUNKS = BLOCK_N / 32;       // epilogue granularity: 32 columns (one TMA store box)
    static constexpr int CHUNK_BYTES = 128 * 64;      // one plane of one chunk: 128 rows x 32 bf16
    static constexpr int SLOT_BYTES = TA * CHUNK_BYTES;  // hi (+ lo)
    // RING: the layer streams epilogue inputs (residual / skip adds); without it the smem goes to operand stages
    static constexpr int RES_BUFS = RING ? 2 : 0;
    static constexpr int RES_DIV = RING ? RES_BUFS : 1;  // RES_BUFS as a divisor (no ring slots are used when RING == 0)
    static constexpr int SMEM_LIMIT = 227 * 1024;
    static constexpr int stages_with(int out_bufs) {
        return (SMEM_LIMIT - 2048 - (out_bufs + RES_BUFS) * SLOT_BYTES) / STAGE_BYTES > 8
                   ? 8
                   : (SMEM_LIMIT - 2048 - (out_bufs + RES_BUFS) * SLOT_BYTES) / STAGE_BYTES;
    }
    // store staging per consumer warpgroup: two slots (chunk c + 1 is written while chunk c is stored) where that costs
    // no operand stage, else one
    static constexpr int OUT_PER_WG = stages_with(4) == stages_with(2) ? 2 : 1;
    static constexpr int OUT_BUFS = 2 * OUT_PER_WG;
    static constexpr int EPI_BYTES = (OUT_BUFS + RES_BUFS) * SLOT_BYTES;
    static constexpr int STAGES = stages_with(OUT_BUFS);
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 2048;  // 1 KB control + 1 KB alignment slack
    static_assert(STAGES >= 2, "need at least a double buffer");
    static_assert(BLOCK_N == 32 || BLOCK_N == 64 || BLOCK_N == 128, "BLOCK_N");
};

// E: element format of activations and weights (common.cuh); ElemF16 requires NTERMS == 1
template <int BLOCK_N, int NTERMS, int RING, class E>
__global__ void __launch_bounds__(384, 1) conv_tc_kernel(const __grid_constant__ ConvParams p) {
    static_assert(!E::F16 || NTERMS == 1, "fp16 operands are single-term");
    using Cfg = ConvCfg<BLOCK_N, NTERMS, RING>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr bool UP = (RING == 2);  // the ring carries low-resolution patches the epilogue interpolates
    extern __shared__ unsigned char smem_raw[];
    // control block at the front, operand ring + epilogue staging 1024-aligned behind it
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_raw);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* rfull_bar = empty_bar + STAGES;
    uint64_t* rempty_bar = rfull_bar + Cfg::RES_BUFS;
    const uint32_t ring = (smem_u32(smem_raw) + 1024u + 1023u) & ~1023u;
    const uint32_t out_stage = ring + STAGES * Cfg::STAGE_BYTES;
    const uint32_t res_stage = out_stage + Cfg::OUT_BUFS * Cfg::SLOT_BYTES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const bool tl = p.dbg_tl != nullptr && blockIdx.x == 0;  // time line of CTA 0: [0] entry [1] set-up done [2] first operands
                                                            // [3] main loop end of the last tile [13] epilogue done [15] exit
    if (tl && threadIdx.x == 0) p.dbg_tl[0] = clock64();
    const int n_extra = RING ? p.has_res + p.n_post : 0;  // epilogue input tensors streamed through the ring
    const bool tma_out = p.out != nullptr;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&p.tmA);
        tma_prefetch_desc(&p.tmB);
        if (p.kchunks2) tma_prefetch_desc(&p.tmA2);
        if (tma_out) tma_prefetch_desc(&p.tmO);
        for (int e = 0; e < n_extra; e++) tma_prefetch_desc(&p.tmR[e]);
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < STAGES; s++) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 4);  // lane 0 of each warp of the consumer warpgroup that used the stage
        }
        for (int s = 0; s < Cfg::RES_BUFS; s++) {
            mbar_init(&rfull_bar[s], 1);
            mbar_init(&rempty_bar[s], 128);  // the consumer warpgroup whose epilogue read the slot
        }
        fence_mbar_init();
    }
    __syncthreads();

    const int num_kb1 = p.kh * p.kw * p.kchunks;
    const int num_kb = num_kb1 + p.kchunks2;
    const int tiles_per_img = p.tiles_x * p.tiles_y;
    const int tw = 1 << p.tw_log2;

    if (tl && threadIdx.x == 0) p.dbg_tl[1] = clock64();
    pdl_wait();     // inputs of this layer are produced by the previous kernel in the stream
    pdl_trigger();  // let the next kernel's CTAs be scheduled onto SMs as they drain (they block in their own wait)
    const long long t_begin = p.dbg ? clock64() : 0;  // CTA lifetime from here: the wait for the previous kernel excluded

    if (warp < 4) {
        // ============================ producer warpgroup ======================
        setmaxnreg_dec<40>();  // two single-lane TMA issuers: their registers go to the consumer warpgroups
        if (warp == 0 && lane == 0) {
            // ---- operand TMA producer: the CTA's tiles in order, num_kb stages each
            int stage = 0;
            uint32_t phase = 0;
            long long w_empty = 0;
            for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
                const int te = p.reverse ? p.total_tiles - 1 - tile : tile;
                const int nt = te % p.n_tiles, mt = te / p.n_tiles;
                const int img = mt / tiles_per_img, r = mt - img * tiles_per_img;
                const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                const int x_in0 = (tx << p.tw_log2) * p.stride - p.pad_x;
                const int y_in0 = ty * p.th * p.stride - p.pad_y;
                for (int kb = 0; kb < num_kb; kb++) {
                    w_empty += mbar_wait_timed(&empty_bar[stage], phase ^ 1u, p.dbg != nullptr);
                    const uint32_t sbase = ring + stage * Cfg::STAGE_BYTES;
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                    const int brow = nt * BLOCK_N;  // rows of the weight tile
                    int kcol, tapc, ax, ay;
                    const CUtensorMap* amap;
                    if (kb < num_kb1) {
                        // taps are visited kx-major (kx outer, ky inner): the accumulation order - hence every result
                        // bit - is the same whichever tile shape computes a layer
                        const int ts = kb / p.kchunks, kc = kb - ts * p.kchunks;
                        const int kx = ts / p.kh, ky = ts - kx * p.kh;
                        amap = &p.tmA, kcol = kc * 64, tapc = ky * p.kw + kx, ax = x_in0 + kx, ay = y_in0 + ky;
                    } else {  // K-concatenated second input (1x1, own stride): weight columns continue after Cin
                        const int kc2 = kb - num_kb1;
                        amap = &p.tmA2, kcol = kc2 * 64, tapc = 0;
                        ax = (tx << p.tw_log2) * p.stride2, ay = ty * p.th * p.stride2;
                    }
                    const int wcol = (kb < num_kb1) ? kcol : (p.kchunks * 64 + kcol);
#pragma unroll
                    for (int t = 0; t < Cfg::TA; t++) {
                        const uint32_t da = sbase + t * Cfg::A_BYTES, db = sbase + Cfg::TA * Cfg::A_BYTES + t * Cfg::B_BYTES;
                        tma_load_5d(da, amap, &full_bar[stage], kcol, ax, ay, img, t);
                        tma_load_4d(db, &p.tmB, &full_bar[stage], wcol, brow, tapc, t);
                    }
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
            }
            if (p.dbg) atomicAdd((unsigned long long*)&p.dbg[ConvDbg::PRODUCER_WAIT_EMPTY], (unsigned long long)w_empty);
        } else if (warp == 1 && lane == 0 && n_extra > 0) {
            // ---- epilogue-input TMA producer: one FIFO of RES_BUFS slots, filled in the CTA's tile order; the epilogues
            // of the two consumer warpgroups take their tiles' entries in that same order
            int cnt = 0;  // fills issued so far
            for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
                const int te = p.reverse ? p.total_tiles - 1 - tile : tile;
                const int nt = te % p.n_tiles, mt = te / p.n_tiles;
                const int img = mt / tiles_per_img, r = mt - img * tiles_per_img;
                const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                for (int c = 0; c < Cfg::CHUNKS; c++) {
                    for (int e = 0; e < n_extra; e++) {
                        const int m = cnt++;
                        const int slot = m % Cfg::RES_DIV;
                        mbar_wait(&rempty_bar[slot], ((uint32_t)(m / Cfg::RES_DIV) & 1u) ^ 1u);
                        int cx = tx << p.tw_log2, cy = ty * p.th;
                        uint32_t bytes = Cfg::SLOT_BYTES;
                        if (UP && e == 0) {  // low-resolution patch under this tile
                            cx = up_src_index(cx, p.up_Wi, p.Wout);
                            cy = up_src_index(cy, p.up_Hi, p.Hout);
                            bytes = (uint32_t)(p.up_pw * p.up_ph * 64 * Cfg::TA);
                        }
                        mbar_arrive_expect_tx(&rfull_bar[slot], bytes);
#pragma unroll
                        for (int t = 0; t < Cfg::TA; t++)
                            tma_load_5d(res_stage + slot * Cfg::SLOT_BYTES + t * Cfg::CHUNK_BYTES, &p.tmR[e],
                                        &rfull_bar[slot], nt * BLOCK_N + c * 32, cx, cy, img, t);
                    }
                }
            }
        }
    } else {
        // ============================ consumer warpgroups: wgmma + epilogue ===
        setmaxnreg_inc<232>();  // 128 fp32 accumulators per thread at BLOCK_N = 128
        const int wg = (warp >> 2) - 1;           // consumer warpgroup 0 / 1: tiles wg, wg + 2, ... of the CTA's list
        const int q4 = lane & 3;                  // column pair 2 q4 of every 8-column group
        const int rw = (warp & 3) * 16 + (lane >> 2);  // this thread's rows: 64 h + rw + 8 i (row half h, i = 0, 1)
        const bool leader = (threadIdx.x & 127) == 0;
        const bool timed = p.dbg != nullptr && leader;
        const uint32_t ob0 = out_stage + (uint32_t)(wg * Cfg::OUT_PER_WG) * Cfg::SLOT_BYTES;  // this warpgroup's staging
        const int n_cta = (p.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;  // tiles of this CTA
        // role counters: operand waits are summed in a register over a tile's main loop (no atomics between its wgmma);
        // epilogue waits go to global memory as they happen (registers are short there in the fused bilinear variants)
        long long* const dc = p.dbg ? p.dbg + ConvDbg::CONS + ConvDbg::CONS_N * wg : nullptr;
        auto tally = [&](int k, long long cycles) {
            if (timed) atomicAdd((unsigned long long*)&dc[k], (unsigned long long)cycles);
        };
        float acc[2][BLOCK_N / 2];  // [row half][wgmma fragment]
        for (int j = wg; j < n_cta; j += 2) {
            const int tile = blockIdx.x + j * gridDim.x;
            const int te = p.reverse ? p.total_tiles - 1 - tile : tile;
            const int nt = te % p.n_tiles, mt = te / p.n_tiles;
            const int img = mt / tiles_per_img, r = mt - img * tiles_per_img;
            const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
            const int n0 = nt * BLOCK_N;

            // ---- main loop, in turn: the operand ring holds the CTA's tiles in order, j * num_kb stages precede this one
            const uint32_t it0 = (uint32_t)j * (uint32_t)num_kb;
            int stage = (int)(it0 % STAGES);
            uint32_t phase = (it0 / STAGES) & 1u;
            if (j > 0) {
                const long long t0 = timed ? clock64() : 0;
                turn_wait(TURN_MAIN, wg);
                tally(ConvDbg::WAIT_ORDER, timed ? clock64() - t0 : 0);
            }
            // one commit group per k-block, the previous k-block's stage is freed once it has retired
            int prev_stage = -1;
            uint32_t w_full = 0;  // per-tile sums fit in 32 bits
            for (int kb = 0; kb < num_kb; kb++) {
                w_full += (uint32_t)mbar_wait_timed(&full_bar[stage], phase, timed);
                if (tl && leader && j == 0 && kb == 0) p.dbg_tl[2] = clock64();
                const uint32_t sbase = ring + stage * Cfg::STAGE_BYTES;
                const uint64_t a0 = wgmma_desc_sw128(sbase);
                const uint64_t b0 = wgmma_desc_sw128(sbase + Cfg::TA * Cfg::A_BYTES);
                constexpr uint64_t A_STEP = (uint64_t)(Cfg::A_BYTES >> 4), B_STEP = (uint64_t)(Cfg::B_BYTES >> 4);
                constexpr uint64_t A_HALF = (uint64_t)((64 * 128) >> 4);  // rows 64..127 of the A tile
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; k++) {  // 4 x k16 per 64-channel k-block; +32 B per step
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const uint64_t ka = a0 + (uint64_t)(k * 2) + h * A_HALF, kbd = b0 + (uint64_t)(k * 2);
                        wgmma_tile<BLOCK_N, E>(acc[h], ka, kbd, (kb | k) != 0);  // a_hi * b_hi
                        if (NTERMS == 3) {
                            wgmma_tile<BLOCK_N, E>(acc[h], ka + A_STEP, kbd, 1u);  // a_lo * b_hi
                            wgmma_tile<BLOCK_N, E>(acc[h], ka, kbd + B_STEP, 1u);  // a_hi * b_lo
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();
                if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
                prev_stage = stage;
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1u;
                }
            }
            if (j + 1 < n_cta) turn_pass(TURN_MAIN, wg ^ 1);  // every wgmma of this tile is issued: the other warpgroup's turn
            tally(ConvDbg::WAIT_FULL, w_full);
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
            if (tl && leader && j == n_cta - 1) p.dbg_tl[3] = clock64();

            // ---- epilogue: this thread's four rows (index 2 h + i), 32 columns (8 values per row) per chunk
            const long long t_epi0 = timed ? clock64() : 0;
            int py[4], px[4];
            bool valid[4];
            long long pix[4];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int row = 64 * (q >> 1) + rw + 8 * (q & 1);
                py[q] = ty * p.th + (row >> p.tw_log2);
                px[q] = (tx << p.tw_log2) + (row & (tw - 1));
                valid[q] = (py[q] < p.Hout) && (px[q] < p.Wout) && (img < p.Nimg);
                pix[q] = ((long long)img * p.Hout + py[q]) * p.Wout + px[q];
            }
            auto row_of = [&](int q) { return 64 * (q >> 1) + rw + 8 * (q & 1); };
            // epilogue inputs arrive through the ring in the order [residual][post1][post2]; this tile's entries follow
            // those of the CTA's j earlier tiles.  The warpgroups take the ring in turns, tile by tile: a parity wait is
            // only sound while the slot's barrier is at most one phase behind, and the other warpgroup may still be reading
            // the previous tile's entries when this one's main loop ends.
            const bool ring_turns = RING != 0 && n_extra > 0;
            if (ring_turns && j > 0) turn_wait(TURN_RING, wg);
            int rcnt = j * Cfg::CHUNKS * n_extra;
            auto ring_wait = [&]() -> uint32_t {
                const int m = rcnt++;
                const int rslot = m % Cfg::RES_DIV;
                tally(ConvDbg::WAIT_RING, mbar_wait_timed(&rfull_bar[rslot], (uint32_t)(m / Cfg::RES_DIV) & 1u, timed));
                return (uint32_t)rslot;
            };
            auto ring_release = [&](uint32_t rslot) {
                // The slot is refilled by TMA (async proxy) while these were generic-proxy reads: without a proxy
                // fence the refill is not ordered after loads that are still in flight.
                fence_proxy_async();
                mbar_arrive(&rempty_bar[rslot]);
            };
            // the fp32 values (low half, high half) of the two channels at byte offset o of a ring slot: hi + lo of the planes,
            // or the widened fp16 pair
            auto ring_f2 = [&](uint32_t rb, uint32_t o) -> float2 {
                if constexpr (E::F16) {
                    const uint32_t w = lds_u32(rb + o);
                    return make_float2(E::lo(w), E::hi(w));
                } else {
                    return planes_to_f2(lds_u32(rb + o), NTERMS == 3 ? lds_u32(rb + Cfg::CHUNK_BYTES + o) : 0u);
                }
            };
            // vv += the fp32 value the next ring slot carries
            auto ring_add = [&](float(&vv)[4][8]) {
                const uint32_t rslot = ring_wait();
                const uint32_t rb = res_stage + rslot * Cfg::SLOT_BYTES;
#pragma unroll
                for (int q = 0; q < 4; q++)
#pragma unroll
                    for (int jj = 0; jj < 4; jj++) {
                        const uint32_t o = sw64_off(row_of(q), jj) + 4 * q4;
                        const float2 rv = ring_f2(rb, o);
                        vv[q][2 * jj] += rv.x;
                        vv[q][2 * jj + 1] += rv.y;
                    }
                ring_release(rslot);
            };
#pragma unroll
            for (int c = 0; c < Cfg::CHUNKS; c++) {
                const int c0 = c * 32;
                float v[4][8];  // [row 2 h + i][8 jj + 2 q4 + e as 2 jj + e]
#pragma unroll
                for (int jj = 0; jj < 4; jj++) {
                    const float2 bia = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + c0 + 8 * jj + 2 * q4));
                    const int f = 4 * (4 * c + jj);  // 8-column group 4 c + jj of the accumulator fragment
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        v[2 * h][2 * jj] = acc[h][f + 0] + bia.x;
                        v[2 * h][2 * jj + 1] = acc[h][f + 1] + bia.y;
                        v[2 * h + 1][2 * jj] = acc[h][f + 2] + bia.x;
                        v[2 * h + 1][2 * jj + 1] = acc[h][f + 3] + bia.y;
                    }
                }
                if (RING == 1 && p.has_res) ring_add(v);
                if (UP) {
                    // bilinear x2 of the low-resolution patch in the ring slot (weights as ATen computes them)
                    const uint32_t rslot = ring_wait();
                    const uint32_t rb = res_stage + rslot * Cfg::SLOT_BYTES;
                    const int oy0 = up_src_index(ty * p.th, p.up_Hi, p.Hout), ox0 = up_src_index(tx << p.tw_log2, p.up_Wi, p.Wout);
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const int pyc = min(py[q], p.Hout - 1), pxc = min(px[q], p.Wout - 1);  // clipped rows are never stored
                        const float sy = up_scale(p.up_Hi, p.Hout) * (float)pyc, sx = up_scale(p.up_Wi, p.Wout) * (float)pxc;
                        const int y0i = (int)sy, x0i = (int)sx;
                        const int y1i = y0i + (y0i < p.up_Hi - 1 ? 1 : 0), x1i = x0i + (x0i < p.up_Wi - 1 ? 1 : 0);
                        const float hy1 = sy - (float)y0i, hy0 = 1.f - hy1, wx1 = sx - (float)x0i, wx0 = 1.f - wx1;
                        const int rr[4] = {(y0i - oy0) * p.up_pw + (x0i - ox0), (y0i - oy0) * p.up_pw + (x1i - ox0),
                                           (y1i - oy0) * p.up_pw + (x0i - ox0), (y1i - oy0) * p.up_pw + (x1i - ox0)};
#pragma unroll
                        for (int jj = 0; jj < 4; jj++) {
                            float2 s[4];
#pragma unroll
                            for (int k = 0; k < 4; k++) {
                                const uint32_t o = sw64_off(rr[k], jj) + 4 * q4;
                                s[k] = ring_f2(rb, o);
                            }
                            v[q][2 * jj] += hy0 * (wx0 * s[0].x + wx1 * s[1].x) + hy1 * (wx0 * s[2].x + wx1 * s[3].x);
                            v[q][2 * jj + 1] += hy0 * (wx0 * s[0].y + wx1 * s[1].y) + hy1 * (wx0 * s[2].y + wx1 * s[3].y);
                        }
                    }
                    ring_release(rslot);
                }
                if (p.relu) {
#pragma unroll
                    for (int q = 0; q < 4; q++)
#pragma unroll
                        for (int e = 0; e < 8; e++) v[q][e] = fmaxf(v[q][e], 0.f);
                }
                for (int e = 0; RING == 1 && e < p.n_post; e++) ring_add(v);  // (relu(..) + skip1) + skip2, left to right
                if (tma_out) {
                    // the staging slot was last read by the store this warpgroup issued OUT_PER_WG chunks ago
                    const uint32_t ob = ob0 + (uint32_t)((((j >> 1) * Cfg::CHUNKS + c) % Cfg::OUT_PER_WG) * Cfg::SLOT_BYTES);
                    if (leader) {
                        const long long t0 = timed ? clock64() : 0;
                        bulk_wait_read<Cfg::OUT_PER_WG - 1>();
                        tally(ConvDbg::WAIT_STAGE, timed ? clock64() - t0 : 0);
                    }
                    // fp16: the clamp-and-count path only runs for a warp that holds a value outside +-65504 (or a NaN)
                    bool sat_warp = false;
                    if constexpr (E::F16) {
                        float m = 0.f;
#pragma unroll
                        for (int q = 0; q < 4; q++)
#pragma unroll
                            for (int e = 0; e < 8; e++) m = E::absmax(m, v[q][e]);
                        sat_warp = __any_sync(0xffffffffu, !(m <= E::MAX));
                    }
                    epi_bar_sync(wg);
                    int n_sat = 0;  // fp16: stored elements of this thread outside +-65504 (clamped)
#pragma unroll
                    for (int q = 0; q < 4; q++)
#pragma unroll
                        for (int jj = 0; jj < 4; jj++) {
                            const float a = v[q][2 * jj], b = v[q][2 * jj + 1];
                            const uint32_t o = sw64_off(row_of(q), jj) + 4 * q4;
                            if constexpr (E::F16) {
                                if (sat_warp) {
                                    int n = 0;
                                    sts_u32(ob + o, E::pack2(E::clamp(a, n), E::clamp(b, n)));
                                    n_sat += valid[q] ? n : 0;  // rows outside the output are never stored
                                } else {
                                    sts_u32(ob + o, E::pack2(a, b));
                                }
                            } else {
                                const uint32_t hw = E::pack2(a, b);  // hi = bf16(v)
                                sts_u32(ob + o, hw);
                                if (NTERMS == 3)  // lo = bf16(v - hi)
                                    sts_u32(ob + Cfg::CHUNK_BYTES + o, E::pack2(a - E::lo(hw), b - E::hi(hw)));
                            }
                        }
                    if constexpr (E::F16)
                        if (sat_warp) saturation_add(p.sat, n_sat);
                    fence_proxy_async();  // generic-proxy smem writes -> visible to the TMA store
                    epi_bar_sync(wg);
                    if (leader) {
#pragma unroll
                        for (int t = 0; t < Cfg::TA; t++)
                            tma_store_5d(&p.tmO, ob + t * Cfg::CHUNK_BYTES, n0 + c0, tx << p.tw_log2, ty * p.th, img, t);
                        bulk_commit();
                    }
                } else {  // fp32 NHWC heads: small tensors, direct stores
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        if (!valid[q]) continue;
#pragma unroll
                        for (int jj = 0; jj < 4; jj++)
                            *reinterpret_cast<float2*>(p.out_f32 + pix[q] * p.Cout + n0 + c0 + 8 * jj + 2 * q4) =
                                make_float2(v[q][2 * jj], v[q][2 * jj + 1]);
                    }
                }
            }
            if (ring_turns && j + 1 < n_cta) turn_pass(TURN_RING, wg ^ 1);  // this tile's ring entries are all released
            tally(ConvDbg::EPILOGUE, timed ? clock64() - t_epi0 : 0);
        }
        if (leader && tma_out) bulk_wait_all();  // stores must be complete before the CTA retires
        // the warpgroup that runs the CTA's last tile finishes last: it closes the CTA's lifetime
        if (leader && wg == ((n_cta - 1) & 1)) {
            if (p.dbg) {
                atomicAdd((unsigned long long*)&p.dbg[ConvDbg::TOTAL], (unsigned long long)(clock64() - t_begin));
                atomicAdd((unsigned long long*)&p.dbg[ConvDbg::CTAS], 1ull);
            }
            if (tl) p.dbg_tl[13] = p.dbg_tl[15] = clock64();
        }
    }
    // no CTA-wide barrier at exit: every TMA load is waited for by a consumer, and each warpgroup leader waits for its
    // own stores, so the roles end independently (the two register budgets never meet again)
}

}  // namespace smapb
