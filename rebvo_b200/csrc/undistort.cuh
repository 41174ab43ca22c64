// undistort.cuh -- the undistortion map of a context (undistort.cu builds it; the gray pass of gray.cu reads it)
#pragma once
#include "common.cuh"

struct rb_undistort {
    rb_ctx *c;
    int4 *inx, *iw;
    int4 *ixy;                   // the taps of inx as x | y << 16, for the strided layout (built with the map; frames of up
                                 // to 65535 x 65535 pixels, rb_pipeline_push_frames_dev)
    uint8_t *tmp_in, *tmp_out;   // staging for the host-pointer entry point
};
