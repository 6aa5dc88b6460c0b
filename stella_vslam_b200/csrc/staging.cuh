// staging.cuh -- host staging of the batched C-ABI entry points.  An entry point lays out its blocks with Layout (inputs, then
// outputs, then device-only scratch), packs the inputs into a StagingArena's pinned mirror, uploads them in one copy, launches,
// downloads the output range in one copy and synchronises before it unpacks.
#pragma once

#include <algorithm>
#include <cstring>

#include "common.cuh"

namespace b200 {

// Offsets of consecutive blocks: every block starts on a 256-byte boundary and takes at least 256 bytes, so no two blocks share
// an offset.  `end` is the total size.
struct Layout {
    size_t end = 0;
    size_t take(size_t bytes) {
        const size_t o = end;
        end += round_up(std::max(bytes, (size_t)1), (size_t)256);
        return o;
    }
    template <typename T>
    size_t take(size_t n) {
        return take(sizeof(T) * n);
    }
};

// A device buffer and its pinned host mirror, owned by a handle; Layout offsets address both.
struct StagingArena {
    unsigned char* d = nullptr;
    unsigned char* h = nullptr;
    size_t d_cap = 0, h_cap = 0;

    // Grows either side to bytes + bytes / 4 + 256.  Waits for st before it frees a buffer that queued work may still read.
    int reserve(size_t dev_bytes, size_t host_bytes, cudaStream_t st) {
        if (dev_bytes > d_cap) {
            B200_CUDA(cudaStreamSynchronize(st));
            if (d) B200_CUDA(cudaFree(d));
            d = nullptr;
            d_cap = 0;
            B200_CUDA(cudaMalloc(&d, dev_bytes + dev_bytes / 4 + 256));
            d_cap = dev_bytes + dev_bytes / 4 + 256;
        }
        if (host_bytes > h_cap) {
            B200_CUDA(cudaStreamSynchronize(st));
            if (h) B200_CUDA(cudaFreeHost(h));
            h = nullptr;
            h_cap = 0;
            B200_CUDA(cudaMallocHost(&h, host_bytes + host_bytes / 4 + 256));
            h_cap = host_bytes + host_bytes / 4 + 256;
        }
        return B200_OK;
    }
    template <typename T = unsigned char>
    T* dev(size_t off) const {
        return reinterpret_cast<T*>(d + off);
    }
    template <typename T = unsigned char>
    T* host(size_t off) const {
        return reinterpret_cast<T*>(h + off);
    }
    void put(size_t off, const void* src, size_t bytes) {
        if (src && bytes) std::memcpy(h + off, src, bytes);
    }
    // [0, bytes) of the mirror to the device
    cudaError_t upload(size_t bytes, cudaStream_t st) { return cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st); }
    // [begin, end) of the device buffer to the mirror; the caller synchronises
    cudaError_t download(size_t begin, size_t end, cudaStream_t st) {
        return cudaMemcpyAsync(h + begin, d + begin, end - begin, cudaMemcpyDeviceToHost, st);
    }
    void release() {
        cudaFree(d);
        if (h) cudaFreeHost(h);
        *this = StagingArena{};
    }
};

}  // namespace b200
