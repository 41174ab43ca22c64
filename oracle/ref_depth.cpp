// TEST INFRASTRUCTURE ONLY -- never linked into, imported by or executed from the product path.
//
// ref_depth.cpp: an extern "C" window onto the UNMODIFIED reference depth_filler (src/visualizer/depth_filler.cpp, compiled
// where it lies by oracle/ref_depth.py into oracle/_ref/libref_depth.so).  ref_depth_fill_net runs the viewer's per-packet
// sequence (src/visualizer/visualizer.cpp:436-440) on n 15-byte net_keyline records:
//   ResetData; FillEdgeData(net_kl, n, {0,0}, thresh_rel_rho, thresh_match_num); InitCoarseFine; Integrate(iter_num);
//   computeDistance(Zeros)
// with depth_filler(cam, {block_w, block_h}, BOUND_NONE) as the viewer constructs it (:303).  Integrate(iter_num) runs
// InitCoarseFine a second time (init_cf = true), as the viewer does.

#include "visualizer/depth_filler.h"
#include <TooN/TooN.h>
#include <cstring>

using namespace rebvo;

extern "C" int ref_depth_fill_net(int w, int h, float ppx, float ppy, float zfx, float zfy, int block_w, int block_h,
                                  double thresh_rel_rho, int thresh_match_num, int iter_num, const void *records, int n,
                                  double *rho, double *s_rho, double *dist, int *fixed, double *min_dist) {
    if (sizeof(net_keyline) != 15) return -1;
    cam_model::rad_tan_distortion kc = {0, 0, 0, 0, 0};
    cam_model cam({ppx, ppy}, {zfx, zfy}, kc, {(u_int)w, (u_int)h});
    depth_filler df(cam, {(u_int)block_w, (u_int)block_h}, depth_filler::BOUND_NONE);
    // the records as the viewer holds them: a net_keyline array inside the packet buffer
    net_keyline *kl = new net_keyline[n > 0 ? n : 1];
    if (n > 0) memcpy(kl, records, (size_t)n * sizeof(net_keyline));
    df.ResetData();
    df.FillEdgeData(kl, n, {0, 0}, thresh_rel_rho, thresh_match_num);
    df.InitCoarseFine();
    df.Integrate(iter_num);
    df.computeDistance(TooN::Zeros);
    delete[] kl;
    const Size2D g = df.gridSize();
    for (u_int i = 0; i < g.w * g.h; i++) {
        rho[i] = df.data[i].rho;
        s_rho[i] = df.data[i].s_rho;
        dist[i] = df.data[i].dist;
        fixed[i] = df.data[i].fixed ? 1 : 0;
    }
    *min_dist = df.GetMinDist();
    return 0;
}
