// TEST INFRASTRUCTURE ONLY -- never linked into, imported by or executed from the product path (the tests are the only
// callers).
//
// ref_pose_graph.cpp: oracle/ref_driver.cpp (the UNMODIFIED reference `REBVO` on a raw frame file), built as a second
// executable (oracle/_ref/ref_rebvo_pg, recipe oracle/build_pose_graph.py) that also writes the pose graph rebvorun saves at
// exit (app/rebvorun/main.cpp:134: cf.poses.saveToFile("poses_list.ps"); pose_graph.cpp:32-40) when the key
// PoseGraphFile=path is given.  The driver is compiled as it is: its one call `cf.CleanUp();` is followed by the save, after
// the three threads have stopped, as in rebvorun.
//
// usage: ref_rebvo_pg frames.bin out.bin PoseGraphFile=poses.ps key=value ...   (other keys: oracle/ref_driver.cpp)

#include "rebvo/rebvo.h"   // (before the macro below: the class declares CleanUp())

#include <cstdio>
#include <string>

static bool ref_save_pose_graph(rebvo::REBVO &cf, const std::string &path) {
    if (path.empty()) return true;
    if (cf.poses.saveToFile(path.c_str())) return true;
    fprintf(stderr, "cannot write %s\n", path.c_str());
    return false;
}

// `cf.CleanUp();` in main() becomes `cf.CleanUp(); if (!ref_save_pose_graph(...)) return 2;` (gets: main's key lookup)
#define CleanUp() CleanUp(); if (!ref_save_pose_graph(cf, gets("PoseGraphFile"))) return 2
#include "ref_driver.cpp"
#undef CleanUp
