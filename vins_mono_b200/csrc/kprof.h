// Per-kernel device timing for bench.py's roofline object: when enabled, every launch group is bracketed by CUDA
// events on the launching stream and waited for (so it serialises the pipeline: profile passes are separate from
// timed passes).  The events are created on the device current at enable(): the owning handle's.
#pragma once
#include <cuda_runtime.h>

#include "cuda_check.h"

namespace vb {

struct KernelProfile {
    static constexpr int MAX_K = 16;
    bool on = false;
    Event a, b;
    double ms[MAX_K] = {};
    int count[MAX_K] = {};
    void enable(bool v) {
        on = v;
        if (v && !a) {
            a.create();
            b.create();
        }
        for (int i = 0; i < MAX_K; i++) ms[i] = 0, count[i] = 0;
    }
    void begin(cudaStream_t s) {
        if (on) cudaEventRecord(a, s);
    }
    void end(int k, cudaStream_t s, int launches = 1) {
        if (!on) return;
        cudaEventRecord(b, s);
        cudaEventSynchronize(b);
        float t = 0;
        cudaEventElapsedTime(&t, a, b);
        ms[k] += t;
        count[k] += launches;
    }
};

}  // namespace vb
