// Offline replay driver: the tracker node loop and the estimator node loop of the reference around the CUDA handles.  A
// session is a list of lanes, each driven by one tracker thread and one estimator thread, and all lanes run concurrently.
// See include/vinsb200/replay.h for the mapping to feature_tracker_node.cpp / estimator_node.cpp.  Pure host code on top of
// the two C ABIs.
#include "vinsb200/replay.h"

#include <cstdio>
#include <cstring>

#include "rotation.h"

#include <atomic>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace {

struct FeatureMsg {
    double stamp = 0;
    std::vector<int> ids;
    std::vector<double> obs;  // n x 7: x y z u v vx vy
    double h2d = 0, d2h = 0;  // tracker traffic of the sequence's images since its previous message
};

struct Step {  // what one image step of a lane's tracker loop produced: at most one feature message per sequence
    std::vector<FeatureMsg> msgs;
    std::vector<char> has;
    long long launches = 0;  // tracker launches of the lane since its previous step
    bool end = false;        // producer is done for this vr_advance call
};

struct Channel {  // bounded queue between the two loops of one lane
    std::mutex m;
    std::condition_variable cv;
    std::deque<Step> q;
    size_t depth = 2;
    void put(Step&& v) {
        std::unique_lock<std::mutex> lk(m);
        cv.wait(lk, [&] { return q.size() < depth; });
        q.push_back(std::move(v));
        cv.notify_all();
    }
    Step get() {
        std::unique_lock<std::mutex> lk(m);
        cv.wait(lk, [&] { return !q.empty(); });
        Step v = std::move(q.front());
        q.pop_front();
        cv.notify_all();
        return v;
    }
};

struct SeqState {
    vt_tracker* trk = nullptr;
    ve_estimator* est = nullptr;
    vr_sequence in{};
    int cursor = 0;           // next image
    bool first_msg = true;    // estimator_node.cpp:167-172
    int imu_k = 0;            // next IMU sample
    double current_time = -1; // estimator_node.cpp:221
    double last_acc[3] = {0, 0, 0}, last_gyr[3] = {0, 0, 0};
    int frames = 0;
    long long launches = 0;   // a lane's kernel launches count on its first sequence: a batch's are not attributable to a member
    double h2d = 0, d2h = 0;
    std::vector<double> traj_t, traj_p;
    struct ReloMsg {  // a /pose_graph/match_points message waiting in relo_buf (estimator_node.cpp:22, 200-206)
        double arrival, frame_stamp;
        int frame_index;
        std::vector<double> match_points;  // x, y, feature id
        double relo_t[3], relo_r[9];
    };
    std::deque<ReloMsg> relo_buf;
    // scratch
    std::vector<float> f_xy, f_id, f_u, f_v, f_vx, f_vy;
    std::vector<double> dt, acc, gyr, states;
};

// A contiguous run of sequences with one queue between its two loops.  The library call of a step is the only thing that
// depends on the mode: a batch lane (vr_open_batch) steps all its sequences through its batch handles in one call, a lane
// of one sequence (vr_open) calls the sequence's own handles.
struct Lane {
    int first = 0, n = 1;  // sequences first .. first + n - 1 of the session
    vt_batch* tb = nullptr;
    ve_batch* eb = nullptr;
    Channel ch;
};

}  // namespace

struct vr_session {
    std::vector<SeqState> seqs;
    std::vector<Lane> lanes;
    std::string error;
    std::mutex err_m;
    std::atomic<int> status{0};
    void fail(int code, const std::string& what) {
        std::lock_guard<std::mutex> lk(err_m);
        if (status.load() == 0) {
            status.store(code);
            error = what;
        }
    }
};

namespace {

// Packs the feature message of the sequence's tracker (estimator_node.cpp:283-302: v = id_of_point + 0.5, feature_id = v / NUM_OF_CAM).
int pack_message(SeqState* q, double stamp, FeatureMsg& msg) {
    const int cap = vt_count(q->trk);
    q->f_xy.resize(2 * (size_t)cap + 2);
    q->f_id.resize(cap + 1);
    q->f_u.resize(cap + 1);
    q->f_v.resize(cap + 1);
    q->f_vx.resize(cap + 1);
    q->f_vy.resize(cap + 1);
    const int n = vt_node_pack(q->trk, cap, q->f_xy.data(), q->f_id.data(), q->f_u.data(), q->f_v.data(), q->f_vx.data(), q->f_vy.data());
    if (n < 0) return n;
    msg.stamp = stamp;
    msg.ids.resize(n);
    msg.obs.resize(7 * (size_t)n);
    for (int k = 0; k < n; k++) {
        msg.ids[k] = (int)(q->f_id[k] + 0.5f);
        double* o = &msg.obs[7 * (size_t)k];
        o[0] = q->f_xy[2 * k];
        o[1] = q->f_xy[2 * k + 1];
        o[2] = 1.0;
        o[3] = q->f_u[k];
        o[4] = q->f_v[k];
        o[5] = q->f_vx[k];
        o[6] = q->f_vy[k];
    }
    return 0;
}

// img_callback for the sequences of one lane.  Every step gives each sequence that still owes published frames its next
// image; the sequences that published hand their feature messages to the estimator loop as one Step.
void tracker_loop(vr_session* s, Lane* L, int n_pub) {
    SeqState* seq = &s->seqs[L->first];
    const int S = L->n;
    std::vector<int> produced(S, 0), active(S), results(S), restarts(S);
    std::vector<const uint8_t*> imgs(S);
    std::vector<double> stamps(S), h2d(S, 0.0), d2h(S, 0.0);
    long long launches = 0;
    while (s->status.load() == 0) {
        bool any = false;
        for (int k = 0; k < S; k++) {
            const SeqState& q = seq[k];
            active[k] = produced[k] < n_pub && q.cursor < q.in.n_images;
            imgs[k] = active[k] ? q.in.images + (size_t)q.cursor * q.in.frame_stride : nullptr;
            stamps[k] = active[k] ? q.in.stamps[q.cursor] : 0;
            any = any || active[k];
        }
        if (!any) break;
        int l = 0;
        if (L->tb) {
            const int rc = vt_batch_node_image(L->tb, active.data(), imgs.data(), seq[0].in.row_stride, stamps.data(),
                                               seq[0].in.images_on_device, results.data(), restarts.data());
            if (rc < 0) {
                s->fail(rc, std::string("tracker batch: ") + vt_batch_last_error(L->tb));
                break;
            }
            vt_batch_last_timing(L->tb, nullptr, &l);
        } else {
            const SeqState& q = seq[0];
            results[0] = q.in.images_on_device ? vt_node_image_device(q.trk, imgs[0], q.in.row_stride, stamps[0], &restarts[0])
                                               : vt_node_image(q.trk, imgs[0], q.in.row_stride, stamps[0], &restarts[0]);
            if (results[0] < 0) {
                s->fail(results[0], std::string("tracker: ") + vt_last_error(q.trk));
                break;
            }
            if (results[0] > 0) vt_last_timing(q.trk, nullptr, &l);  // a gated-out image leaves the handle's timing stale
        }
        launches += l;
        Step step;
        step.msgs.resize(S);
        step.has.assign(S, 0);
        bool any_msg = false;
        for (int k = 0; k < S; k++) {
            if (!active[k]) continue;
            SeqState& q = seq[k];
            q.cursor++;
            if (results[k] > 0) {
                double a = 0, b = 0;
                vt_last_traffic(q.trk, &a, &b);
                h2d[k] += a;
                d2h[k] += b;
            }
            if (results[k] != 2) continue;
            FeatureMsg& msg = step.msgs[k];
            const int rc = pack_message(&q, stamps[k], msg);
            if (rc < 0) {
                s->fail(rc, L->tb ? "tracker batch: vt_node_pack" : "tracker: vt_node_pack");
                break;
            }
            msg.h2d = h2d[k];
            msg.d2h = d2h[k];
            h2d[k] = d2h[k] = 0;
            step.has[k] = 1;
            produced[k]++;
            any_msg = true;
        }
        if (any_msg) {
            step.launches = launches;
            launches = 0;
            L->ch.put(std::move(step));
        }
    }
    Step fin;
    fin.end = true;
    L->ch.put(std::move(fin));
}

void imu_one(SeqState* q, int k, double img_t) {
    const double t = q->in.imu_t[k];
    const double* a = q->in.acc + 3 * (size_t)k;
    const double* g = q->in.gyr + 3 * (size_t)k;
    if (t <= img_t) {
        if (q->current_time < 0) q->current_time = t;
        const double dt = t - q->current_time;
        q->current_time = t;
        for (int c = 0; c < 3; c++) {
            q->last_acc[c] = a[c];
            q->last_gyr[c] = g[c];
        }
        q->dt.push_back(dt);
    } else {
        const double dt_1 = img_t - q->current_time, dt_2 = t - img_t;
        q->current_time = img_t;
        const double w1 = dt_2 / (dt_1 + dt_2), w2 = dt_1 / (dt_1 + dt_2);
        for (int c = 0; c < 3; c++) {
            q->last_acc[c] = w1 * q->last_acc[c] + w2 * a[c];
            q->last_gyr[c] = w1 * q->last_gyr[c] + w2 * g[c];
        }
        q->dt.push_back(dt_1);
    }
    for (int c = 0; c < 3; c++) {
        q->acc.push_back(q->last_acc[c]);
        q->gyr.push_back(q->last_gyr[c]);
    }
}

// getMeasurements + the dt / interpolation rules of process() for one image stamp: fills q->dt / acc / gyr
void collect_imu(SeqState* q, double stamp) {
    q->dt.clear();
    q->acc.clear();
    q->gyr.clear();
    while (q->imu_k < q->in.n_imu && q->in.imu_t[q->imu_k] < stamp) {
        imu_one(q, q->imu_k, stamp);
        q->imu_k++;
    }
    if (q->imu_k < q->in.n_imu) imu_one(q, q->imu_k, stamp);  // used, but stays in the buffer
}

// process(): "set relocalization frame" (estimator_node.cpp:266-291): every message that has arrived by now is popped, the LAST
// one is handed to setReloFrame.
void apply_relo(SeqState* q, double now) {
    const SeqState::ReloMsg* last = nullptr;
    size_t n_pop = 0;
    for (auto& m : q->relo_buf) {
        if (m.arrival > now) break;
        last = &m;
        n_pop++;
    }
    if (last)
        ve_set_relo_frame(q->est, last->frame_stamp, last->frame_index, (int)(last->match_points.size() / 3), last->match_points.data(),
                          last->relo_t, last->relo_r);
    for (size_t k = 0; k < n_pop; k++) q->relo_buf.pop_front();
}

// process() for the sequences of one lane.  Per sequence with a message: the first message is dropped, the others get
// their IMU samples up to stamp + td and their relocalisation message.  An IMU failure ends the step there.  Then one
// processImage call serves the whole step, and every sequence it processed adds a trajectory row.
void estimator_loop(vr_session* s, Lane* L) {
    SeqState* seq = &s->seqs[L->first];
    const int S = L->n;
    std::vector<int> active(S), n(S), status(S);
    std::vector<const int*> ids(S);
    std::vector<const double*> obs(S);
    std::vector<double> stamps(S);
    for (;;) {
        Step step = L->ch.get();
        if (step.end) break;
        if (s->status.load() != 0) continue;  // keep draining so that the producer can finish
        seq[0].launches += step.launches;
        bool any = false;
        for (int k = 0; k < S; k++) {
            active[k] = 0;
            n[k] = 0;
            ids[k] = nullptr;
            obs[k] = nullptr;
            stamps[k] = 0;
            if (!step.has[k]) continue;
            SeqState& q = seq[k];
            const FeatureMsg& msg = step.msgs[k];
            q.h2d += msg.h2d;
            q.d2h += msg.d2h;
            if (q.first_msg) {  // estimator_node.cpp:167-172
                q.first_msg = false;
                q.frames++;
                continue;
            }
            double td = 0;  // img_t = stamp + estimator.td in getMeasurements and process() (estimator_node.cpp:106-126, 232-265)
            ve_get_states(q.est, q.states.data(), &td);
            collect_imu(&q, msg.stamp + td);
            const int rc = q.dt.empty() ? 0 : ve_process_imu_batch(q.est, (int)q.dt.size(), q.dt.data(), q.acc.data(), q.gyr.data());
            if (rc < 0) {
                s->fail(rc, std::string("estimator: ") + ve_last_error(q.est));
                break;
            }
            apply_relo(&q, msg.stamp);
            active[k] = 1;
            n[k] = (int)msg.ids.size();
            ids[k] = msg.ids.data();
            obs[k] = msg.obs.data();
            stamps[k] = msg.stamp;
            any = true;
        }
        if (s->status.load() != 0 || !any) continue;
        int rc, l = 0;
        if (L->eb) {
            rc = ve_batch_process_image(L->eb, active.data(), n.data(), ids.data(), obs.data(), stamps.data(), status.data());
            if (rc < 0) s->fail(rc, std::string("estimator batch: ") + ve_batch_last_error(L->eb));
            else ve_batch_last_timing(L->eb, nullptr, &l);
        } else {
            rc = ve_process_image(seq[0].est, n[0], ids[0], obs[0], stamps[0]);
            if (rc < 0) s->fail(rc, std::string("estimator: ") + ve_last_error(seq[0].est));
            else ve_last_timing(seq[0].est, nullptr, &l);
        }
        if (rc < 0) continue;
        seq[0].launches += l;
        for (int k = 0; k < S; k++) {
            if (!active[k]) continue;
            SeqState& q = seq[k];
            double a = 0, b = 0;
            ve_last_traffic(q.est, &a, &b);
            q.h2d += a;
            q.d2h += b;
            q.frames++;
            int info[10];
            double costs[2];
            if (ve_info(q.est, info, costs) == 0 && info[0] == 1) {
                ve_get_states(q.est, q.states.data(), nullptr);
                const double* newest = &q.states[16 * (size_t)info[1]];  // frame_count == WINDOW_SIZE: the newest frame
                q.traj_t.push_back(stamps[k]);
                q.traj_p.insert(q.traj_p.end(), newest, newest + 3);
            }
        }
    }
}

// The argument checks and the set-up vr_open and vr_open_batch share: a SeqState per sequence, and one lane of all the
// sequences for a batch (tb, eb) or a lane per sequence.
int open_session(int n_seq, vt_tracker* const* trk, ve_estimator* const* est, const vr_sequence* seqs, vt_batch* tb, ve_batch* eb,
                 vr_session** out) {
    for (int k = 0; k < n_seq; k++)
        if (!trk[k] || !est[k] || !seqs[k].images || !seqs[k].stamps || (seqs[k].n_imu > 0 && !seqs[k].imu_t)) return -1;
    auto* s = new vr_session;
    s->seqs = std::vector<SeqState>(n_seq);
    for (int k = 0; k < n_seq; k++) {
        SeqState& q = s->seqs[k];
        q.trk = trk[k];
        q.est = est[k];
        q.in = seqs[k];
        q.states.assign(16 * (size_t)(ve_window_size(est[k]) + 1), 0.0);
    }
    s->lanes = std::vector<Lane>(tb ? 1 : n_seq);
    for (size_t l = 0; l < s->lanes.size(); l++) {
        Lane& L = s->lanes[l];
        L.first = (int)l;
        L.n = tb ? n_seq : 1;
        L.tb = tb;
        L.eb = eb;
    }
    *out = s;
    return 0;
}

}  // namespace

extern "C" {

int vr_open_batch(vt_batch* trackers, ve_batch* estimators, const vr_sequence* seqs, vr_session** out) {
    if (!trackers || !estimators || !seqs || !out) return -1;
    const int n_seq = vt_batch_size(trackers);
    if (n_seq <= 0 || n_seq != ve_batch_size(estimators)) return -1;
    std::vector<vt_tracker*> trk(n_seq);
    std::vector<ve_estimator*> est(n_seq);
    for (int k = 0; k < n_seq; k++) {
        if (seqs[k].row_stride != seqs[0].row_stride || seqs[k].images_on_device != seqs[0].images_on_device) return -1;
        trk[k] = vt_batch_member(trackers, k);
        est[k] = ve_batch_member(estimators, k);
    }
    return open_session(n_seq, trk.data(), est.data(), seqs, trackers, estimators, out);
}

int vr_open(int n_seq, vt_tracker* const* trackers, ve_estimator* const* estimators, const vr_sequence* seqs, vr_session** out) {
    if (n_seq <= 0 || !trackers || !estimators || !seqs || !out) return -1;
    return open_session(n_seq, trackers, estimators, seqs, nullptr, nullptr, out);
}

void vr_close(vr_session* s) { delete s; }

const char* vr_last_error(const vr_session* s) { return s ? s->error.c_str() : "null session"; }

int vr_advance(vr_session* s, int n_pub) {
    if (!s || n_pub < 0) return -1;
    if (s->status.load() != 0) return s->status.load();
    std::vector<int> before(s->seqs.size());
    std::vector<std::thread> threads;
    for (size_t k = 0; k < s->seqs.size(); k++) before[k] = s->seqs[k].frames;
    for (Lane& L : s->lanes) {
        threads.emplace_back(tracker_loop, s, &L, n_pub);
        threads.emplace_back(estimator_loop, s, &L);
    }
    for (auto& t : threads) t.join();
    if (s->status.load() != 0) return s->status.load();
    int total = 0;
    for (size_t k = 0; k < s->seqs.size(); k++) total += s->seqs[k].frames - before[k];
    return total;
}

int vr_debug_imu_batches(int n_imu, const double* imu_t, const double* acc, const double* gyr, int n_stamps, const double* stamps,
                         int cap, int* counts, double* dt, double* acc_out, double* gyr_out) {
    if (n_imu < 0 || n_stamps < 0 || !imu_t || !acc || !gyr || !stamps || !counts) return -1;
    SeqState q;
    q.in.n_imu = n_imu;
    q.in.imu_t = imu_t;
    q.in.acc = acc;
    q.in.gyr = gyr;
    int total = 0;
    for (int k = 0; k < n_stamps; k++) {
        collect_imu(&q, stamps[k]);
        counts[k] = (int)q.dt.size();
        for (size_t i = 0; i < q.dt.size(); i++, total++) {
            if (total >= cap) return -2;
            if (dt) dt[total] = q.dt[i];
            for (int c = 0; c < 3; c++) {
                if (acc_out) acc_out[3 * total + c] = q.acc[3 * i + c];
                if (gyr_out) gyr_out[3 * total + c] = q.gyr[3 * i + c];
            }
        }
    }
    return total;
}

// ---- node shells, remainder ------------------------------------------------------------------------------------------
}  // extern "C"

struct vr_propagator {  // the globals of estimator_node.cpp:21-40
    double latest_time = 0;
    vb::Vec3 tmp_P, tmp_V, tmp_Ba, tmp_Bg, acc_0, gyr_0, g;
    vb::Quat tmp_Q;
    bool init_imu = true;
};

namespace {
void prop_one(vr_propagator* p, double t, const double* a, const double* w) {
    if (p->init_imu) {
        p->latest_time = t;
        p->init_imu = false;
        return;
    }
    const double dt = t - p->latest_time;
    p->latest_time = t;
    const vb::Vec3 acc(a[0], a[1], a[2]), gyr(w[0], w[1], w[2]);
    const vb::Vec3 un_acc_0 = vb::qrot(p->tmp_Q, p->acc_0 - p->tmp_Ba) - p->g;
    const vb::Vec3 un_gyr = 0.5 * (p->gyr_0 + gyr) - p->tmp_Bg;
    p->tmp_Q = vb::qmul(p->tmp_Q, vb::deltaQ(un_gyr * dt));
    const vb::Vec3 un_acc_1 = vb::qrot(p->tmp_Q, acc - p->tmp_Ba) - p->g;
    const vb::Vec3 un_acc = 0.5 * (un_acc_0 + un_acc_1);
    p->tmp_P = p->tmp_P + dt * p->tmp_V + 0.5 * dt * dt * un_acc;
    p->tmp_V = p->tmp_V + dt * un_acc;
    p->acc_0 = acc;
    p->gyr_0 = gyr;
}
void prop_out(const vr_propagator* p, double* o) {
    if (!o) return;
    o[0] = p->tmp_P.x; o[1] = p->tmp_P.y; o[2] = p->tmp_P.z;
    o[3] = p->tmp_Q.w; o[4] = p->tmp_Q.x; o[5] = p->tmp_Q.y; o[6] = p->tmp_Q.z;
    o[7] = p->tmp_V.x; o[8] = p->tmp_V.y; o[9] = p->tmp_V.z;
}
}  // namespace

extern "C" {

vr_propagator* vr_prop_create(void) { return new vr_propagator; }
void vr_prop_destroy(vr_propagator* p) { delete p; }

int vr_prop_predict(vr_propagator* p, double t, const double* acc, const double* gyr, double* out10) {
    if (!p || !acc || !gyr) return -1;
    prop_one(p, t, acc, gyr);
    prop_out(p, out10);
    return 0;
}

int vr_prop_update(vr_propagator* p, double current_time, const double* P3, const double* Q, const double* V3, const double* Ba3,
                   const double* Bg3, const double* acc0, const double* gyr0, const double* g3, int n, const double* t, const double* acc,
                   const double* gyr) {
    if (!p || !P3 || !Q || !V3 || !Ba3 || !Bg3 || !acc0 || !gyr0 || !g3 || n < 0 || (n && (!t || !acc || !gyr))) return -1;
    p->latest_time = current_time;
    p->tmp_P = vb::Vec3(P3[0], P3[1], P3[2]);
    p->tmp_Q = vb::Quat(Q[0], Q[1], Q[2], Q[3]);
    p->tmp_V = vb::Vec3(V3[0], V3[1], V3[2]);
    p->tmp_Ba = vb::Vec3(Ba3[0], Ba3[1], Ba3[2]);
    p->tmp_Bg = vb::Vec3(Bg3[0], Bg3[1], Bg3[2]);
    p->acc_0 = vb::Vec3(acc0[0], acc0[1], acc0[2]);
    p->gyr_0 = vb::Vec3(gyr0[0], gyr0[1], gyr0[2]);
    p->g = vb::Vec3(g3[0], g3[1], g3[2]);
    for (int k = 0; k < n; k++) prop_one(p, t[k], acc + 3 * k, gyr + 3 * k);
    return 0;
}

int vr_prop_update_from_estimator(vr_propagator* p, const ve_estimator* e, double current_time, int n, const double* t, const double* acc,
                                  const double* gyr) {
    if (!p || !e) return -1;
    int info[10];
    if (ve_info(e, info, nullptr) != 0) return -1;
    const int W = ve_window_size(e);
    std::vector<double> st(16 * (size_t)(W + 1), 0.0);
    double imu0[9];
    if (ve_get_states(e, st.data(), nullptr) != 0 || ve_get_latest_imu(e, imu0, imu0 + 3, imu0 + 6) != 0) return -1;
    const double* s = &st[16 * (size_t)W];
    return vr_prop_update(p, current_time, s, s + 3, s + 7, s + 10, s + 13, imu0, imu0 + 3, imu0 + 6, n, t, acc, gyr);
}

int vr_format_result_row(double stamp, const double* P3, const double* Q, const double* V3, char* buf, int cap) {
    if (!P3 || !Q || !V3 || !buf || cap <= 0) return -1;
    // ofstream with ios::fixed: precision 0 for the nanosecond stamp, 5 for the rest, a comma after every field
    const int n = std::snprintf(buf, (size_t)cap, "%.0f,%.5f,%.5f,%.5f,%.5f,%.5f,%.5f,%.5f,%.5f,%.5f,%.5f,\n", stamp * 1e9, P3[0], P3[1], P3[2],
                                Q[0], Q[1], Q[2], Q[3], V3[0], V3[1], V3[2]);
    return n < cap ? n : -1;
}

int vr_decode_pointcloud(int n, const float* xyz, const float* id_of_point, const float* u_of_point, const float* v_of_point,
                         const float* velocity_x, const float* velocity_y, int* feature_ids, int* camera_ids, double* obs7) {
    if (n < 0 || (n && (!xyz || !id_of_point || !u_of_point || !v_of_point || !velocity_x || !velocity_y || !feature_ids || !obs7))) return -1;
    const int NUM_OF_CAM = 1;
    for (int i = 0; i < n; i++) {
        const int v = (int)(id_of_point[i] + 0.5f);
        feature_ids[i] = v / NUM_OF_CAM;
        if (camera_ids) camera_ids[i] = v % NUM_OF_CAM;
        if (xyz[3 * i + 2] != 1.0f) return -1;  // ROS_ASSERT(z == 1)
        double* o = obs7 + 7 * (size_t)i;
        o[0] = xyz[3 * i];
        o[1] = xyz[3 * i + 1];
        o[2] = xyz[3 * i + 2];
        o[3] = u_of_point[i];
        o[4] = v_of_point[i];
        o[5] = velocity_x[i];
        o[6] = velocity_y[i];
    }
    return n;
}

int vr_decode_relo_message(int n, const float* xyz, const float* channel0_values8, double* match_points, double* relo_t3, double* relo_r9,
                           int* frame_index) {
    if (n < 0 || (n && (!xyz || !match_points)) || !channel0_values8 || !relo_t3 || !relo_r9) return -1;
    for (int i = 0; i < n; i++) {  // u_v_id = (points[i].x, points[i].y, points[i].z)
        match_points[3 * i] = xyz[3 * i];
        match_points[3 * i + 1] = xyz[3 * i + 1];
        match_points[3 * i + 2] = xyz[3 * i + 2];
    }
    const float* c = channel0_values8;
    for (int k = 0; k < 3; k++) relo_t3[k] = c[k];
    // Quaterniond relo_q(values[3], values[4], values[5], values[6]) = (w, x, y, z); toRotationMatrix() does not normalise
    const vb::Mat3 R = vb::Quat(c[3], c[4], c[5], c[6]).R();
    std::memcpy(relo_r9, R.m, sizeof(R.m));
    if (frame_index) *frame_index = (int)c[7];
    return n;
}

int vr_queue_relo(vr_session* s, int seq, double arrival_stamp, double frame_stamp, int frame_index, int n, const double* match_points,
                  const double* relo_t3, const double* relo_r9) {
    if (!s || seq < 0 || seq >= (int)s->seqs.size() || n < 0 || (n && !match_points) || !relo_t3 || !relo_r9) return -1;
    SeqState::ReloMsg m;
    m.arrival = arrival_stamp;
    m.frame_stamp = frame_stamp;
    m.frame_index = frame_index;
    m.match_points.assign(match_points, match_points + 3 * (size_t)n);
    std::memcpy(m.relo_t, relo_t3, sizeof(m.relo_t));
    std::memcpy(m.relo_r, relo_r9, sizeof(m.relo_r));
    auto& buf = s->seqs[seq].relo_buf;  // kept in arrival order
    auto it = buf.end();
    while (it != buf.begin() && (it - 1)->arrival > arrival_stamp) --it;
    buf.insert(it, std::move(m));
    return 0;
}

int vr_stats(const vr_session* s, int seq, int* frames, long long* launches, double* h2d_bytes, double* d2h_bytes) {
    if (!s || seq < 0 || seq >= (int)s->seqs.size()) return -1;
    const SeqState& q = s->seqs[seq];
    if (frames) *frames = q.frames;
    if (launches) *launches = q.launches;
    if (h2d_bytes) *h2d_bytes = q.h2d;
    if (d2h_bytes) *d2h_bytes = q.d2h;
    return 0;
}

int vr_trajectory(const vr_session* s, int seq, int cap, double* stamps, double* positions3) {
    if (!s || seq < 0 || seq >= (int)s->seqs.size()) return -1;
    const SeqState& q = s->seqs[seq];
    const int n = (int)q.traj_t.size();
    for (int k = 0; k < n && k < cap; k++) {
        if (stamps) stamps[k] = q.traj_t[k];
        if (positions3)
            for (int c = 0; c < 3; c++) positions3[3 * k + c] = q.traj_p[3 * (size_t)k + c];
    }
    return n;
}

}  // extern "C"
