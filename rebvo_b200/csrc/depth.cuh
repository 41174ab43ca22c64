// depth.cuh -- the viewer's per-frame depth grid (depth.cu): geometry of one fill and the enqueue entry the pipeline uses
#pragma once
#include "common.cuh"

#define RB_DEPTH_MAX_LEVELS 24
#define RB_DEPTH_THREADS 1024
#define RB_DEPTH_STREAMS 8        // side streams of the pipeline's fills (pipeline.cu)

// depth_filler(cam, {block_w, block_h}, BOUND_NONE) on the context's camera, with FillEdgeData's / Integrate's parameters
struct DepthGeom {
    int gw, gh, bw, bh;           // grid = frame / block in integer division (depth_filler.cpp:31)
    double thresh_rel_rho;
    int thresh_match_num, iter_num;
    float ppx, ppy;
    double zfm;                   // cam_model::zfm, (zfx + zfy) / 2 in float
    // InitCoarseFine's tile levels, coarsest first: tile size, tiles per row / column, index of the level's first tile
    int nlev, ntiles;
    int lsx[RB_DEPTH_MAX_LEVELS], lsy[RB_DEPTH_MAX_LEVELS], lnx[RB_DEPTH_MAX_LEVELS], lny[RB_DEPTH_MAX_LEVELS],
        loff[RB_DEPTH_MAX_LEVELS];
    int in_smem;                  // 1: the grid lives in dynamic shared memory, 0: in the global workspace
};

struct DepthPlan {
    DepthGeom g;
    size_t grid_bytes;            // rho, s_rho, tile means, fixed bits, tile flags
    size_t dyn_smem;              // grid_bytes when it fits in shared memory, else 0
    size_t cells_bytes;           // gw * gh rb_depth_cell records followed by min_dist, rounded up to 256
};

// RB_ERR_ARG for a block < 1 or larger than the frame, iter_num < 0
int rb_depth_plan(rb_ctx *c, const rb_depth_params *p, DepthPlan *out);
// global workspace of one fill over at most kcap records
size_t rb_depth_ws_bytes(const DepthPlan &pl, int kcap);
// one fill CTA on c->stream.  Records: rec_pp ? rec_pp[0] + rec_ofs : rec; their number: kn_p ? *kn_p : kn (at most kcap).
// Cells (then min_dist): out_pp ? out_pp[1] + out_ofs : out.
int rb_depth_fill_enqueue(rb_ctx *c, const DepthPlan &pl, const unsigned char *const *rec_pp, size_t rec_ofs,
                          const unsigned char *rec, const int *kn_p, int kn, int kcap, void *ws,
                          unsigned char *const *out_pp, size_t out_ofs, rb_depth_cell *out);
