// Error handling of the CUDA calls behind the C ABI: a failing call records "<call>: <CUDA error string>" in owner->err
// (what the *_last_error entry points return) and makes the calling function return `ret`.
#pragma once
#include <cuda_runtime.h>

#include <string>

#define VB_CUDA_CHECK(owner, ret, call)                                          \
    do {                                                                         \
        const cudaError_t vb_err_ = (call);                                      \
        if (vb_err_ != cudaSuccess) {                                            \
            (owner)->err = std::string(#call) + ": " + cudaGetErrorString(vb_err_); \
            return ret;                                                          \
        }                                                                        \
    } while (0)
