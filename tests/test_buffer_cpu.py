"""The owning device / pinned buffer of the host code (csrc/decode_host.h), compiled into a small host program against a
stand-in for the CUDA runtime's allocation calls and last-error state, so that it runs the same with or without a device
or a driver: a failed grow leaves the buffer empty with capacity 0, returns the error and leaves nothing in the last-error
state for the next launch check to report; grow re-allocates only above the capacity; moves hand the memory over; and
each kind is freed once, by its own call."""
import shutil
import subprocess

import pytest

from smap_b200 import build

PROGRAM = r"""
#include <stdio.h>
#include <stdlib.h>

#include <set>

#include "decode_host.h"

// Allocations of up to 1 MiB succeed (in host memory); larger ones fail as an out-of-memory cudaMalloc does.
static cudaError_t g_last = cudaSuccess;
static std::set<void*> g_dev, g_pinned;  // live allocations of each kind
static cudaError_t alloc(std::set<void*>& live, void** p, size_t n) {
    if (n > (1 << 20)) return g_last = cudaErrorMemoryAllocation;
    *p = malloc(n);
    live.insert(*p);
    return cudaSuccess;
}
static cudaError_t release(std::set<void*>& live, void* p) {
    if (!live.erase(p)) return g_last = cudaErrorInvalidValue;  // freed twice, or by the other kind's call
    free(p);
    return cudaSuccess;
}
extern "C" {
cudaError_t cudaMalloc(void** p, size_t n) { return alloc(g_dev, p, n); }
cudaError_t cudaMallocHost(void** p, size_t n) { return alloc(g_pinned, p, n); }
cudaError_t cudaFree(void* p) { return release(g_dev, p); }
cudaError_t cudaFreeHost(void* p) { return release(g_pinned, p); }
cudaError_t cudaGetLastError(void) {
    const cudaError_t e = g_last;
    g_last = cudaSuccess;
    return e;
}
}

#define CHECK(c)                                                 \
    if (!(c)) {                                                  \
        printf("%s: line %d: %s\n", kind, __LINE__, #c);         \
        return 1;                                                \
    }

template <typename T, bool Pinned>
static int check(const char* kind, const std::set<void*>& live) {
    {
        smapb::Buffer<T, Pinned> b;
        CHECK(b.grow(100) == cudaSuccess && b.get() && b.capacity() == 100 && live.size() == 1);
        T* const p = b;
        CHECK(b.grow(100) == cudaSuccess && b.grow(50) == cudaSuccess && b.get() == p && b.capacity() == 100);
        CHECK(b.grow((size_t)1 << 30) == cudaErrorMemoryAllocation);
        CHECK(b.get() == nullptr && b.capacity() == 0 && live.empty());
        CHECK(cudaGetLastError() == cudaSuccess);
        CHECK(b.grow(10) == cudaSuccess);
        smapb::Buffer<T, Pinned> c(std::move(b));
        CHECK(b.get() == nullptr && b.capacity() == 0 && c.get() && c.capacity() == 10 && live.size() == 1);
        smapb::Buffer<T, Pinned> d;
        CHECK(d.grow(20) == cudaSuccess && live.size() == 2);
        c = std::move(d);
        CHECK(d.get() == nullptr && c.capacity() == 20 && live.size() == 1);
    }
    CHECK(live.empty() && cudaGetLastError() == cudaSuccess);
    return 0;
}

int main() {
    if (check<float, false>("device", g_dev) || check<int, true>("pinned", g_pinned)) return 1;
    printf("ok\n");
    return 0;
}
"""


def test_owning_buffer_against_a_stand_in_runtime(tmp_path):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not found")
    src, exe = tmp_path / "buffer.cpp", tmp_path / "buffer"
    src.write_text(PROGRAM)
    subprocess.run(["nvcc", "-std=c++17", "-cudart", "none", "-I", build.CSRC, str(src), "-o", str(exe)], check=True)
    p = subprocess.run([str(exe)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0 and p.stdout == "ok\n", p.stdout
