// owners.hpp -- move-only owners of the host side's CUDA resources, freed by their destructors with the resource's
// device selected by the caller.  Kernel parameter structs (BatchBuffers, TrainBuffers, ModelTiles) keep raw pointers.
#pragma once
#include <cstddef>
#include <utility>
#include <vector>

#include <cuda_runtime.h>

namespace nnb {

// A handle released by Destroy(h), e.g. a stream or an event; a null handle is skipped.
template <typename H, auto Destroy>
class Owner {
  public:
    Owner() = default;
    Owner(Owner&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    Owner& operator=(Owner&& o) noexcept {
        reset(std::exchange(o.h_, nullptr));
        return *this;
    }
    ~Owner() { reset(); }
    void reset(H h = nullptr) {
        if (h_) Destroy(h_);
        h_ = h;
    }
    H* put() {  // for the creator call that writes the new handle
        reset();
        return &h_;
    }
    operator H() const { return h_; }

  private:
    H h_ = nullptr;
};

using Stream = Owner<cudaStream_t, cudaStreamDestroy>;
using Event = Owner<cudaEvent_t, cudaEventDestroy>;
using PinnedMem = Owner<void*, cudaFreeHost>;

// One device allocation and its size in bytes.
class DeviceMem {
  public:
    DeviceMem() = default;
    DeviceMem(DeviceMem&& o) noexcept { *this = std::move(o); }
    DeviceMem& operator=(DeviceMem&& o) noexcept {
        p_ = std::move(o.p_);
        bytes_ = std::exchange(o.bytes_, 0);
        return *this;
    }
    cudaError_t alloc(size_t bytes) {  // frees the old allocation first
        reset();
        void* q = nullptr;
        const cudaError_t e = cudaMalloc(&q, bytes);
        if (e != cudaSuccess) return e;
        p_.reset(q);
        bytes_ = bytes;
        return e;
    }
    void reset() {
        p_.reset();
        bytes_ = 0;
    }
    template <typename T = void>
    T* get() const { return static_cast<T*>(static_cast<void*>(p_)); }
    size_t bytes() const { return bytes_; }

  private:
    Owner<void*, cudaFree> p_;
    size_t bytes_ = 0;
};

// A device array of `count` elements at *p, owned by a new last entry of *mem.
template <typename T>
cudaError_t dalloc(std::vector<DeviceMem>* mem, T** p, size_t count) {
    mem->emplace_back();
    const cudaError_t e = mem->back().alloc(count * sizeof(T));
    *p = mem->back().get<T>();
    return e;
}

}  // namespace nnb
