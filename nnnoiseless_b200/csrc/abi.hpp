// abi.hpp -- the host conventions every C-ABI entry point follows (DESIGN.md §1):
//   - an error sets rnnoise_last_error() and the entry point returns -1 (NULL for a creator);
//   - an entry point runs with its handle's device selected and gives the caller its current device back;
//   - a creator opens its device by open_device's rules;
//   - a list of stream indices is checked by check_streams before anything runs;
//   - device work is ordered after the caller's CUDA stream, and the caller's stream continues after it (without a
//     stream, the call returns when the work has finished).
#pragma once
#include <string>

#include <cuda_runtime.h>

namespace nnb {

// Sets rnnoise_last_error() to `what`, followed by ": <CUDA error text>" when e is an error; returns -1.
int fail(const std::string& what, cudaError_t e = cudaSuccess);
// Adds n kernels to rnnoise_kernel_launches().
void count_launches(int n);

// A failed CUDA call returns fail("<call>", its error) from the enclosing function.
#define CK(call)                                         \
    do {                                                 \
        cudaError_t e__ = (call);                        \
        if (e__ != cudaSuccess) return fail(#call, e__); \
    } while (0)

// Selects `dev` for the rest of the scope and then gives the caller its current device back (a multi-GPU host thread,
// e.g. PyTorch with tensors elsewhere, must not find its device switched behind its back).
struct DeviceGuard {
    int prev = -1, want = -1;
    cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int dev) : want(dev) {
        err = cudaGetDevice(&prev);
        if (err == cudaSuccess && prev != dev) err = cudaSetDevice(dev);
    }
    ~DeviceGuard() {
        if (prev >= 0 && prev != want) cudaSetDevice(prev);
    }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// The rest of the enclosing function runs on device `dev`.
#define ON_DEVICE(dev)                \
    DeviceGuard guard__(dev);         \
    if (guard__.err != cudaSuccess) return fail("cudaSetDevice", guard__.err)

// The device of a new handle: `device`, or the current device when it is negative.  Fails without a usable device and
// for an index past the last device.  Selects nothing.
int open_device(int device, int* chosen);

// Checks n stream indices of a handle (a `holder`) of `total` streams: in range and none twice.  streams NULL stands for
// 0..n-1.
int check_streams(int total, const int* streams, int n, const char* holder);
inline int stream_of(const int* streams, int r) { return streams ? streams[r] : r; }

// Orders s after the work queued so far on the caller's stream `us` (NULL: nothing to wait for), through event ev.
int wait_for_caller(cudaStream_t s, cudaStream_t us, cudaEvent_t ev);
// The caller's stream `us` continues after the work queued so far on s, through event ev; without one, s is
// synchronised.
int resume_caller(cudaStream_t s, cudaStream_t us, cudaEvent_t ev);

}  // namespace nnb
