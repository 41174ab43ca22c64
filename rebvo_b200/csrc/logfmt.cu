// logfmt.cu -- on-disk formats of the reference's third thread (SURVEY.md 8(f) rank 4), host code:
//   trajectory file (TrayFile)   rebvo_third_t.cpp:311      "t x y z  qx qy qz qw " per frame, std::scientific, precision 18,
//                                                           TooN vector streaming (a blank after every element, vector.hh:670-677),
//                                                           quaternion = util::LieRot2Quaternion(PoseLie) (toon_util.h:63-72)
//   m-file log (LogFile)         rebvo_third_t.cpp:265-281  the per-frame records that are functions of the pose / map
//                                                           (Kp, RKp, Rot, Vel, t, dt, i, Pose, Pos, K, KLN; std::scientific,
//                                                           precision 16, :151); the IMU, stereo and wall-clock records of that
//                                                           block (:283-305) are not part of the hot path's output
//   pose graph (poses_list.ps)   pose_graph.cpp:32-40       binary OdometryMeas records, written by rebvorun at exit
// Text is produced from rb_nav records and the pose graph from rb_odometry records, so a consumer of the GPU pipeline writes the
// same files the reference writes.
#include "common.cuh"
#include <cmath>
#include <cstddef>
#include <cstdio>

namespace {
struct Out {
    char *buf;
    size_t cap, len;
    bool overflow;
    void put(const char *s, int n) {
        if (n < 0) return;
        if (len + (size_t)n <= cap && buf) memcpy(buf + len, s, n);
        else overflow = true;
        len += n;
    }
    void f18(double v) {   // std::scientific << std::setprecision(18)
        char t[64];
        put(t, snprintf(t, sizeof(t), "%.18e", v));
    }
    void g(double v) {     // a_log << std::scientific << std::setprecision(16) (rebvo_third_t.cpp:151)
        char t[64];
        put(t, snprintf(t, sizeof(t), "%.16e", v));
    }
    void s(const char *str) { put(str, (int)strlen(str)); }
    void i(long long v) {
        char t[32];
        put(t, snprintf(t, sizeof(t), "%lld", v));
    }
};
}   // namespace

extern "C" int rb_nav_format_trajectory(const rb_nav *nav, int n, double time_scale, char *buf, size_t cap, size_t *written) {
    if (!nav || n < 0 || time_scale == 0) return RB_ERR_ARG;
    Out o{buf, cap, 0, false};
    for (int k = 0; k < n; k++) {
        const rb_nav &r = nav[k];
        // LieRot2Quaternion: q = {W / |W| * sin(|W| / 2), cos(|W| / 2)}
        const double *W = r.PoseLie;
        const double angle = sqrt(W[0] * W[0] + W[1] * W[1] + W[2] * W[2]);
        double q[4] = {0, 0, 0, 0};
        if (angle > 0) {
            const double sh = sin(angle / 2);
            for (int j = 0; j < 3; j++) q[j] = W[j] / angle * sh;
        }
        q[3] = cos(angle / 2);
        o.f18(r.t / time_scale);
        o.s(" ");
        for (int j = 0; j < 3; j++) {
            o.f18(r.Pos[j]);
            o.s(" ");
        }
        o.s(" ");
        for (int j = 0; j < 4; j++) {
            o.f18(q[j]);
            o.s(" ");
        }
        o.s("\n");
    }
    if (written) *written = o.len;
    return o.overflow ? RB_ERR_ARG : RB_OK;
}

static void mat3(Out &o, const char *name, long long idx, const double *M) {
    o.s(name);
    o.s("(");
    o.i(idx);
    o.s(",:,:)=[");
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) {
            o.g(M[r * 3 + c]);
            o.s(c < 2 ? "," : (r < 2 ? ";" : "];\n"));
        }
}
static void vec3(Out &o, const char *name, long long idx, const double *v) {
    o.s(name);
    o.s("(");
    o.i(idx);
    o.s(",:)=[");
    o.g(v[0]);
    o.s(",");
    o.g(v[1]);
    o.s(",");
    o.g(v[2]);
    o.s("];\n");
}
static void scal(Out &o, const char *name, long long idx, double v) {
    o.s(name);
    o.s("(");
    o.i(idx);
    o.s(",:)=");
    o.g(v);
    o.s(";\n");
}

// first_index: a_log_inx of the first record (the reference counts from 1); frame_id0: p_id of the first record
extern "C" int rb_nav_format_log(const rb_nav *nav, int n, long long first_index, long long frame_id0, char *buf, size_t cap,
                                 size_t *written) {
    if (!nav || n < 0) return RB_ERR_ARG;
    Out o{buf, cap, 0, false};
    for (int k = 0; k < n; k++) {
        const rb_nav &r = nav[k];
        const long long idx = first_index + k;
        scal(o, "Kp_cv", idx, r.Kp);
        scal(o, "RKp_cv", idx, r.RKp);
        mat3(o, "Rot_cv", idx, r.Rot);
        vec3(o, "Vel_cv", idx, r.Vel);
        scal(o, "t_cv", idx, r.t);
        scal(o, "dt_cv", idx, r.dt);
        o.s("i_cv(");
        o.i(idx);
        o.s(",:)=");
        o.i(frame_id0 + k);
        o.s(";\n");
        mat3(o, "Pose_cv", idx, r.Pose);
        vec3(o, "Pos_cv", idx, r.Pos);
        scal(o, "K_cv", idx, r.K);
        o.s("KLN_cv(");
        o.i(idx);
        o.s(",:)=");
        o.i(r.kn);
        o.s(";\n");
    }
    if (written) *written = o.len;
    return o.overflow ? RB_ERR_ARG : RB_OK;
}

// pose graph file (poses_list.ps, app/rebvorun/main.cpp:134): pose_graph::saveToFile writes a uint count, then
// OdometryMeas::dumpToFile per record: every vector / matrix element as a raw double (matrices row by row), KF_ID as a raw int.
// rb_odometry holds the 81 doubles in that order without padding, so a record is two contiguous pieces.
static_assert(offsetof(rb_odometry, KF_ID) == 81 * sizeof(double), "rb_odometry: doubles of OdometryMeas, packed");
extern "C" int rb_odometry_format_pose_graph(const rb_odometry *r, int n, void *buf, size_t cap, size_t *written) {
    if (n < 0 || (!r && n > 0)) return RB_ERR_ARG;
    Out o{static_cast<char *>(buf), cap, 0, false};
    uint32_t count = 0;
    for (int k = 0; k < n; k++) count += r[k].tracked != 0;
    o.put(reinterpret_cast<const char *>(&count), sizeof(count));
    for (int k = 0; k < n; k++)
        if (r[k].tracked) {
            o.put(reinterpret_cast<const char *>(r[k].relPosPose), (int)offsetof(rb_odometry, KF_ID));
            o.put(reinterpret_cast<const char *>(&r[k].KF_ID), sizeof(int32_t));
        }
    if (written) *written = o.len;
    return o.overflow ? RB_ERR_ARG : RB_OK;
}
