// depth.cuh -- the viewer's per-frame depth grid and its dense image (depth.cu): geometry of one fill and one image pass,
// and the enqueue entries the pipeline uses
#pragma once
#include "common.cuh"

#define RB_DEPTH_MAX_LEVELS 24
#define RB_DEPTH_THREADS 1024
#define RB_DEPTH_STREAMS 8        // side streams of the pipeline's fills (pipeline.cu)
#define RB_DEPTH_IMG_THREADS 256

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

// the image pass over the w x h frame: depth_filler::getImgRho at every pixel of the grid of a fill
struct DepthImgGeom {
    int w, h, gw, gh, bw, bh;
    int planes;                   // 1: rho, 2: rho and s_rho
    int in_smem;                  // 1: each CTA stages the grid as float pairs in dynamic shared memory, 0: reads it in place
};
struct DepthImgPlan {
    DepthImgGeom g;
    size_t dyn_smem;              // gw * gh * 8 when the grid fits in shared memory, else 0
    int ctas;
};

// RB_ERR_ARG for a block < 1 or larger than the frame, iter_num < 0
int rb_depth_plan(rb_ctx *c, const rb_depth_params *p, DepthPlan *out);
// global workspace of one fill over at most kcap records
size_t rb_depth_ws_bytes(const DepthPlan &pl, int kcap);
// where in that workspace a fill with keep_final leaves the final (rho, s_rho) of every cell (gw * gh double pairs)
double2 *rb_depth_ws_final(const DepthPlan &pl, int kcap, void *ws);
// one fill CTA on c->stream.  Records: rec_pp ? rec_pp[0] + rec_ofs : rec; their number: kn_p ? *kn_p : kn (at most kcap).
// Cells (then min_dist): out_pp ? out_pp[1] + out_ofs : out.  keep_final: also the cells' (rho, s_rho) in the workspace.
int rb_depth_fill_enqueue(rb_ctx *c, const DepthPlan &pl, const unsigned char *const *rec_pp, size_t rec_ofs,
                          const unsigned char *rec, const int *kn_p, int kn, int kcap, void *ws,
                          unsigned char *const *out_pp, size_t out_ofs, rb_depth_cell *out, bool keep_final);
// the image pass of a fill's grid with `planes` planes (1 or 2) on the context's frame size
int rb_depth_image_plan(rb_ctx *c, const DepthGeom &g, int planes, DepthImgPlan *out);
// the image pass on c->stream.  Cell i: rho = src[i * stride], s_rho = src[i * stride + 1] (device memory).  Planes: rho at
// out_pp ? out_pp[0] + out_ofs (bytes) : out, s_rho plane_floats floats after it; both must start on 16 bytes.
int rb_depth_image_enqueue(rb_ctx *c, const DepthImgPlan &ip, const double *src, int stride, float *const *out_pp,
                           size_t out_ofs, float *out, size_t plane_floats);
