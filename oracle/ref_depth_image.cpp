// TEST INFRASTRUCTURE ONLY -- never linked into, imported by or executed from the product path.
//
// ref_depth_image.cpp: an extern "C" window onto the UNMODIFIED reference depth_filler (src/visualizer/depth_filler.cpp,
// compiled where it lies by oracle/ref_depth_image.py into oracle/_ref/libref_depth_image.so) that samples the grid at
// every pixel of the frame with the header's own depth_filler::getImgRho(x, y, &s_rho), integer pixel coordinates passed
// as float (as gl_viewer::drawFillerUnc does).  Two ways to the grid:
//   ref_depth_image_net    the viewer's per-packet sequence (src/visualizer/visualizer.cpp:436-440) on n 15-byte
//                          net_keyline records, as oracle/ref_depth.cpp runs it;
//   ref_depth_image_cells  rho / s_rho written straight into the public depth_filler::data, for crafted grids.
// Outputs: getImgRho's double return and s_rho, row-major h x w.

#include "visualizer/depth_filler.h"
#include <TooN/TooN.h>
#include <cstring>

using namespace rebvo;

static void sample(depth_filler &df, int w, int h, double *rho, double *s_rho) {
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            double s = 0;
            rho[(size_t)y * w + x] = df.getImgRho((float)x, (float)y, &s);
            s_rho[(size_t)y * w + x] = s;
        }
}

extern "C" int ref_depth_image_net(int w, int h, float ppx, float ppy, float zfx, float zfy, int block_w, int block_h,
                                   double thresh_rel_rho, int thresh_match_num, int iter_num, const void *records, int n,
                                   double *rho, double *s_rho) {
    if (sizeof(net_keyline) != 15) return -1;
    cam_model::rad_tan_distortion kc = {0, 0, 0, 0, 0};
    cam_model cam({ppx, ppy}, {zfx, zfy}, kc, {(u_int)w, (u_int)h});
    depth_filler df(cam, {(u_int)block_w, (u_int)block_h}, depth_filler::BOUND_NONE);
    net_keyline *kl = new net_keyline[n > 0 ? n : 1];
    if (n > 0) memcpy(kl, records, (size_t)n * sizeof(net_keyline));
    df.ResetData();
    df.FillEdgeData(kl, n, {0, 0}, thresh_rel_rho, thresh_match_num);
    df.InitCoarseFine();
    df.Integrate(iter_num);
    df.computeDistance(TooN::Zeros);
    delete[] kl;
    sample(df, w, h, rho, s_rho);
    return 0;
}

extern "C" int ref_depth_image_cells(int w, int h, int block_w, int block_h, const double *cell_rho,
                                     const double *cell_s_rho, double *rho, double *s_rho) {
    cam_model::rad_tan_distortion kc = {0, 0, 0, 0, 0};
    cam_model cam({w / 2.0f, h / 2.0f}, {500.0f, 500.0f}, kc, {(u_int)w, (u_int)h});
    depth_filler df(cam, {(u_int)block_w, (u_int)block_h}, depth_filler::BOUND_NONE);
    df.ResetData();
    const Size2D g = df.gridSize();
    for (u_int i = 0; i < g.w * g.h; i++) {
        df.data[i].rho = cell_rho[i];
        df.data[i].s_rho = cell_s_rho[i];
    }
    sample(df, w, h, rho, s_rho);
    return 0;
}
