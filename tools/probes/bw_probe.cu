// Read-bandwidth ceilings on this GPU for the two access paths the association kernels use (tools only):
//   (1) LDG.128 streaming (grid-stride float4 loads, U loads in flight per thread)
//   (2) cp.async.bulk (UBLKCP) global -> shared, one persistent CTA per SM, double-buffered, chunk size C
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probes/bw_probe tools/probes/bw_probe.cu && tools/probes/bw_probe
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int U>
__global__ void ldg_stream(const float4* __restrict__ src, size_t n4, float* out) {
    float acc = 0.f;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride * U) {
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; u++) v[u] = (i + u * stride < n4) ? __ldg(src + i + u * stride) : make_float4(0, 0, 0, 0);
#pragma unroll
        for (int u = 0; u < U; u++) acc += v[u].x + v[u].y + v[u].z + v[u].w;
    }
    if (acc == 123.456f) *out = acc;
}

__global__ void __launch_bounds__(128, 1) bulk_stream(const char* __restrict__ src, size_t bytes_per_cta, uint32_t buf_bytes,
                                                      uint32_t chunk, float* out) {
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem);  // [2]
    unsigned char* buf[2] = {smem + 128, smem + 128 + buf_bytes};
    const char* base = src + (size_t)blockIdx.x * bytes_per_cta;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 2; i++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar[i])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int n_fill = (int)(bytes_per_cta / buf_bytes);
    auto issue = [&](int f) {
        if (threadIdx.x < 32) {
            const int b = f & 1;
            if (threadIdx.x == 0)
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar[b])), "r"(buf_bytes) : "memory");
            __syncwarp();
            for (uint32_t off = threadIdx.x * chunk; off < buf_bytes; off += 32 * chunk)
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                                 smem_u32(buf[b] + off)),
                             "l"(base + (size_t)f * buf_bytes + off), "r"(chunk), "r"(smem_u32(&bar[b]))
                             : "memory");
        }
    };
    issue(0);
    if (n_fill > 1) issue(1);
    float acc = 0.f;
    for (int f = 0; f < n_fill; f++) {
        const int b = f & 1;
        const uint32_t parity = (f >> 1) & 1;
        if (threadIdx.x < 32) {
            uint32_t ok = 0;
            while (!ok)
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                             : "=r"(ok) : "r"(smem_u32(&bar[b])), "r"(parity) : "memory");
        }
        __syncthreads();
        acc += reinterpret_cast<float*>(buf[b])[threadIdx.x];
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (f + 2 < n_fill) issue(f + 2);
    }
    if (acc == 123.456f) *out = acc;
}

int main() {
    const size_t bytes = (size_t)132 * 213 * 1024 * 48;  // ~1.5 GB
    char* src;
    float* out;
    cudaMalloc(&src, bytes);
    cudaMalloc(&out, 4);
    cudaMemset(src, 1, bytes);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    auto report = [&](const char* name, float ms, size_t b) { printf("%-46s %8.3f ms  %7.0f GB/s\n", name, ms, b / ms * 1e-6); };
    for (int rep = 0; rep < 2; rep++) {
        float ms;
        cudaEventRecord(e0);
        ldg_stream<4><<<132 * 8, 256>>>((const float4*)src, bytes / 16, out);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        if (rep) report("LDG.128 x4 in flight, 132*8 CTAs x 256", ms, bytes);
        cudaEventRecord(e0);
        ldg_stream<8><<<132 * 8, 256>>>((const float4*)src, bytes / 16, out);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        if (rep) report("LDG.128 x8 in flight, 132*8 CTAs x 256", ms, bytes);
        const uint32_t bufs[3] = {106496, 65536, 32768};
        const uint32_t chunks[4] = {2048, 8192, 16384, 32768};
        for (uint32_t bb : bufs)
            for (uint32_t ch : chunks) {
                if (bb % ch) continue;
                const size_t per_cta = (bytes / 132) / bb * bb;
                cudaFuncSetAttribute(bulk_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 + 2 * bb);
                cudaEventRecord(e0);
                bulk_stream<<<132, 128, 128 + 2 * bb>>>(src, per_cta, bb, ch, out);
                cudaEventRecord(e1);
                cudaEventSynchronize(e1);
                cudaEventElapsedTime(&ms, e0, e1);
                char name[96];
                snprintf(name, sizeof name, "UBLKCP 1 CTA/SM, 2 x %u KB buffers, %u KB chunks", bb / 1024, ch / 1024);
                if (rep) report(name, ms, per_cta * 132);
            }
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
