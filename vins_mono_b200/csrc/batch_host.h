// What the batched handle families of the C ABI share (vt_batch of vt_tracker, ve_batch of ve_estimator, vp_batch of
// vp_graph), host code only.  A batch owns its S members; a stand-alone handle is a batch of one, marked so that
// destroying its only member destroys it.  Each family's entry points are thin wrappers over the functions below.
//
// The first part is plain C++ (tests/hostlib/batch_host_check.cpp builds it with g++ over a dummy member type); the
// destroy and profile part at the end needs the CUDA runtime and is compiled by nvcc only.
#pragma once
#include <memory>
#include <string>
#include <vector>

namespace vb {

template <class Batch>
struct MemberBase {
    Batch* batch = nullptr;
    int member = 0;   // index in batch->members
    std::string err;  // this member's last error
};

template <class Member>
struct BatchBase {
    int S = 0;
    bool standalone = false;  // made by the family's *_create: destroyed with its only member
    std::string err;          // the batch's last error
    std::vector<std::unique_ptr<Member>> members;
};

template <class B>
int batch_size(const B* b, int invalid) {
    return b ? b->S : invalid;
}

template <class B>
auto batch_member(B* b, int k) -> decltype(b->members[0].get()) {
    return (b && k >= 0 && k < b->S) ? b->members[k].get() : nullptr;
}

template <class B>
const char* batch_last_error(const B* b) {
    return b ? b->err.c_str() : "null batch";
}

// A member's own text when it has one, else its batch's: a batch call that failed for all its members leaves the
// members' texts empty.
template <class M>
const char* last_error(const M* m) {
    if (!m) return "null handle";
    return m->err.empty() ? m->batch->err.c_str() : m->err.c_str();
}

// The status of a batch step: ok, or the first failing member's status, with "member k: <its text>" as the batch's text.
template <class B>
int roll_up(B* b, int ok) {
    for (int k = 0; k < b->S; k++) {
        const auto& m = *b->members[k];
        if (m.status != ok) {
            b->err = "member " + std::to_string(k) + ": " + m.err;
            return m.status;
        }
    }
    return ok;
}

// Per-handle calls that advance a handle are for stand-alone handles; a member of an explicit batch advances through
// its batch's call.  Returns 0 for a stand-alone handle, else `invalid` with `text` (naming that call) as m's error.
template <class M>
int refuse_member(M* m, int invalid, const char* text) {
    if (m->batch->standalone) return 0;
    m->err = text;
    return invalid;
}

// *_create: a batch of one from create(cfg, 1, &b), marked stand-alone; *out is its member.
template <class Cfg, class B, class M>
int create_standalone(int (*create)(const Cfg*, int, B**), const Cfg* cfg, M** out, int invalid) {
    if (!cfg || !out) return invalid;
    *out = nullptr;
    B* b = nullptr;
    const int rc = create(cfg, 1, &b);
    if (rc) return rc;
    b->standalone = true;
    *out = b->members[0].get();
    return 0;
}

// *_destroy: destroys a stand-alone handle's batch; a member of an explicit batch goes with its batch.
template <class M, class B>
void destroy_standalone(M* m, void (*destroy)(B*)) {
    if (m && m->batch->standalone) destroy(m->batch);
}

template <class B>
int kernel_times(const B* b, double* ms, int* count, int n, int invalid) {
    if (!b) return invalid;
    for (int k = 0; k < n; k++) {
        if (ms) ms[k] = b->prof.ms[k];
        if (count) count[k] = b->prof.count[k];
    }
    return 0;
}

}  // namespace vb

#ifdef __CUDACC__
#include "cuda_check.h"

namespace vb {

// *_batch_destroy: on the batch's device, drain() waits for the batch's streams and stops its host work; then the
// members go, then the batch's own buffers, streams and events.
template <class B, class Drain>
void destroy_batch(B* b, Drain drain) {
    if (!b) return;
    cudaSetDevice(b->cfg.device);
    drain();
    b->members.clear();
    delete b;
}

template <class B>
int set_profile(B* b, int on, int invalid, int cuda_error) {
    if (!b) return invalid;
    VB_CUDA_CHECK(b, cuda_error, cudaSetDevice(b->cfg.device));
    b->prof.enable(on != 0);
    return 0;
}

}  // namespace vb
#endif
