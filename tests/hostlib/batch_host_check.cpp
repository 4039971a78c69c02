// The CUDA-free part of vins_mono_b200/csrc/batch_host.h over a dummy member type, compiled with g++ by
// tests/test_batch_host.py.  Each check_* entry returns its failure count and writes the first failure into msg.
#include <cstdio>
#include <cstring>
#include <string>

#include "batch_host.h"

namespace {

int g_member_dtors = 0, g_batch_dtors = 0;

struct Batch;
struct Member : vb::MemberBase<Batch> {
    int status = 0;
    ~Member() { g_member_dtors++; }
};
struct Profile {
    double ms[16] = {};
    int count[16] = {};
};
struct Batch : vb::BatchBase<Member> {
    Profile prof;
    ~Batch() { g_batch_dtors++; }
};
struct Config {
    int fail = 0;
};

constexpr int OK = 0, INVALID = -1;

int create(const Config* cfg, int n, Batch** out) {
    *out = nullptr;
    if (cfg->fail) return cfg->fail;
    Batch* b = new Batch;
    b->S = n;
    for (int k = 0; k < n; k++) {
        b->members.emplace_back(new Member);
        b->members[k]->batch = b;
        b->members[k]->member = k;
    }
    *out = b;
    return OK;
}

void destroy(Batch* b) {
    b->members.clear();
    delete b;
}

struct Checks {
    char* msg;
    int cap, failures = 0;
    void operator()(bool ok, const char* what, int line) {
        if (!ok && failures++ == 0) std::snprintf(msg, cap, "line %d: %s", line, what);
    }
};
#define CHECK(c, cond) c(cond, #cond, __LINE__)

bool same(const char* a, const char* b) { return std::strcmp(a, b) == 0; }

}  // namespace

extern "C" int check_member_bounds(char* msg, int cap) {
    Checks c{msg, cap};
    Config cfg;
    Batch* b = nullptr;
    create(&cfg, 3, &b);
    CHECK(c, vb::batch_size(b, INVALID) == 3);
    CHECK(c, vb::batch_size<Batch>(nullptr, INVALID) == INVALID);
    for (int k = 0; k < 3; k++) {
        Member* m = vb::batch_member(b, k);
        CHECK(c, m == b->members[k].get() && m->batch == b && m->member == k);
    }
    CHECK(c, vb::batch_member(b, -1) == nullptr);
    CHECK(c, vb::batch_member(b, 3) == nullptr);
    CHECK(c, vb::batch_member<Batch>(nullptr, 0) == nullptr);
    destroy(b);
    return c.failures;
}

extern "C" int check_last_error(char* msg, int cap) {
    Checks c{msg, cap};
    Batch* b = nullptr;
    Config cfg;
    create(&cfg, 2, &b);
    Member* m = b->members[1].get();
    CHECK(c, same(vb::last_error(m), ""));
    b->err = "batch text";
    CHECK(c, same(vb::last_error(m), "batch text"));  // the member has no text of its own
    m->err = "member text";
    CHECK(c, same(vb::last_error(m), "member text"));
    CHECK(c, same(vb::last_error(b->members[0].get()), "batch text"));
    CHECK(c, same(vb::batch_last_error(b), "batch text"));
    CHECK(c, same(vb::last_error<Member>(nullptr), "null handle"));
    CHECK(c, same(vb::batch_last_error<Batch>(nullptr), "null batch"));
    destroy(b);
    return c.failures;
}

extern "C" int check_roll_up(char* msg, int cap) {
    Checks c{msg, cap};
    Batch* b = nullptr;
    Config cfg;
    create(&cfg, 4, &b);
    b->err = "before";
    CHECK(c, vb::roll_up(b, OK) == OK);
    CHECK(c, b->err == "before");  // nothing failed: the batch's text stays
    b->members[1]->status = -4;
    b->members[1]->err = "capacity";
    b->members[3]->status = -3;
    b->members[3]->err = "cuda";
    CHECK(c, vb::roll_up(b, OK) == -4);
    CHECK(c, b->err == "member 1: capacity");
    CHECK(c, b->members[1]->err == "capacity" && b->members[3]->err == "cuda");
    b->members[1]->status = OK;
    CHECK(c, vb::roll_up(b, OK) == -3);
    CHECK(c, b->err == "member 3: cuda");
    destroy(b);
    return c.failures;
}

extern "C" int check_refuse_member(char* msg, int cap) {
    Checks c{msg, cap};
    Config cfg;
    Batch* b = nullptr;
    create(&cfg, 2, &b);
    Member* m = b->members[0].get();
    CHECK(c, vb::refuse_member(m, INVALID, "use the batch call") == INVALID);
    CHECK(c, m->err == "use the batch call");
    destroy(b);
    Member* s = nullptr;
    vb::create_standalone(create, &cfg, &s, INVALID);
    s->err = "kept";
    CHECK(c, vb::refuse_member(s, INVALID, "use the batch call") == 0);
    CHECK(c, s->err == "kept");
    vb::destroy_standalone(s, destroy);
    return c.failures;
}

// Destroying a member destroys its batch (and the member) only when the batch is stand-alone.
extern "C" int check_standalone(char* msg, int cap) {
    Checks c{msg, cap};
    Config cfg;
    Member* s = nullptr;
    CHECK(c, vb::create_standalone(create, &cfg, &s, INVALID) == OK);
    CHECK(c, s && s->batch->standalone && s->batch->S == 1 && s == s->batch->members[0].get());
    g_member_dtors = g_batch_dtors = 0;
    vb::destroy_standalone(s, destroy);
    CHECK(c, g_member_dtors == 1 && g_batch_dtors == 1);

    Batch* b = nullptr;
    create(&cfg, 2, &b);
    g_member_dtors = g_batch_dtors = 0;
    vb::destroy_standalone(b->members[0].get(), destroy);
    vb::destroy_standalone<Member, Batch>(nullptr, destroy);
    CHECK(c, g_member_dtors == 0 && g_batch_dtors == 0);
    destroy(b);
    CHECK(c, g_member_dtors == 2 && g_batch_dtors == 1);

    Member marker;
    Member* out = &marker;
    CHECK(c, vb::create_standalone(create, static_cast<const Config*>(nullptr), &out, INVALID) == INVALID);
    Member** no_out = nullptr;
    CHECK(c, vb::create_standalone(create, &cfg, no_out, INVALID) == INVALID);
    Config failing{-2};
    CHECK(c, vb::create_standalone(create, &failing, &out, INVALID) == -2 && out == nullptr);
    return c.failures;
}

extern "C" int check_kernel_times(char* msg, int cap) {
    Checks c{msg, cap};
    Config cfg;
    Batch* b = nullptr;
    create(&cfg, 1, &b);
    for (int k = 0; k < 16; k++) b->prof.ms[k] = 0.5 * k, b->prof.count[k] = k;
    double ms[8] = {};
    int count[8] = {};
    CHECK(c, vb::kernel_times(b, ms, count, 6, INVALID) == 0);
    CHECK(c, ms[5] == 2.5 && count[5] == 5 && ms[6] == 0 && count[6] == 0);
    CHECK(c, vb::kernel_times(b, nullptr, count, 8, INVALID) == 0 && count[7] == 7);
    CHECK(c, vb::kernel_times<Batch>(nullptr, ms, count, 8, INVALID) == INVALID);
    destroy(b);
    return c.failures;
}
