// TEST INFRASTRUCTURE ONLY -- never linked into, imported by or executed from the product path.
//
// ref_live_imu.cpp: the UNMODIFIED reference `REBVO` in live IMU mode (ImuMode=1: ImuGrabber(CircBufferSize, SampleTime),
// rebvo.cpp:249-260), driven like app/rebvorun/main_custom_cam_example.cpp:52-82 and the ROS nodelet
// (rebvo_nodelet.cpp:140): before it hands over frame k it calls REBVO::pushIMU for every sample up to that frame's time and
// the first sample past it, so FirstThr's GrabAndIntegrate (rebvo_first_t.cpp:293-302) finds the frame's window covered or
// waits for the next frame's samples.
//
// Inputs: the raw frame file of oracle/ref_driver.cpp and a raw sample file (ImuSamples=path: float64 rows
// {t, gyro xyz, accel xyz}).  Output: the records of oracle/ref_driver.cpp (refapi.OUTREC, read by refapi.run_full_rebvo) and
// its JSON line.  Linked once against the compiled reference (ref_live_imu) and once against the shim (shim_live_imu).
//
// usage: ref_live_imu frames.bin out.bin ImuSamples=imu.bin [SampleTime=0.005] [CircBufferSize=1000] [key=value ...]

#include "rebvo/rebvo.h"
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <thread>
#include <vector>

using namespace rebvo;

struct OutRec {   // == oracle/ref_driver.cpp's record
    double t, Pos[3], PoseLie[3], Pose[9], Vel[3], RotLie[3];
    double dtp0, dtp1, K, Kp, s_rho_p;
    int kn, matches, est_ok, p_id;
    double Rot[9], RKp, dt;
};
static std::vector<OutRec> g_out;
static volatile int g_ncb = 0;

static bool callback(PipeBuffer &pb) {
    OutRec r;
    memset(&r, 0, sizeof(r));
    r.t = pb.t;
    for (int i = 0; i < 3; i++) {
        r.Pos[i] = pb.nav.Pos[i];
        r.PoseLie[i] = pb.nav.PoseLie[i];
        r.Vel[i] = pb.nav.Vel[i];
        r.RotLie[i] = pb.nav.RotLie[i];
        for (int j = 0; j < 3; j++) {
            r.Pose[i * 3 + j] = pb.nav.Pose(i, j);
            r.Rot[i * 3 + j] = pb.nav.Rot(i, j);
        }
    }
    r.dtp0 = pb.dtp0;
    r.dtp1 = pb.dtp1;
    r.K = pb.K;
    r.Kp = pb.Kp;
    r.s_rho_p = pb.s_rho_p;
    r.kn = pb.ef->KNum();
    r.matches = pb.ef->NumMatches();
    r.est_ok = pb.EstimationOK;
    r.p_id = pb.p_id;
    r.RKp = pb.RKp;
    r.dt = pb.dt;
    g_out.push_back(r);
    g_ncb++;
    return true;
}

static bool read_all(const char *path, std::vector<unsigned char> &out) {
    FILE *f = fopen(path, "rb");
    if (!f) return false;
    unsigned char buf[1 << 16];
    size_t k;
    while ((k = fread(buf, 1, sizeof(buf), f)) > 0) out.insert(out.end(), buf, buf + k);
    fclose(f);
    return true;
}

int main(int argc, char **argv) {
    if (argc < 3) {
        fprintf(stderr, "usage: %s frames.bin out.bin ImuSamples=imu.bin [key=value ...]\n", argv[0]);
        return 2;
    }
    std::map<std::string, double> kv;
    std::map<std::string, std::string> skv;
    for (int i = 3; i < argc; i++) {
        char *eq = strchr(argv[i], '=');
        if (eq) {
            kv[std::string(argv[i], eq - argv[i])] = atof(eq + 1);
            skv[std::string(argv[i], eq - argv[i])] = std::string(eq + 1);
        }
    }
    auto get = [&](const char *k, double d) { return kv.count(k) ? kv[k] : d; };

    std::vector<unsigned char> raw;
    if (!read_all(argv[1], raw) || raw.size() < 12) {
        fprintf(stderr, "cannot read %s\n", argv[1]);
        return 2;
    }
    int hdr[3];
    memcpy(hdr, raw.data(), 12);
    const int W = hdr[0], H = hdr[1], NF = hdr[2];
    const size_t fb = (size_t)W * H * 3;
    if (raw.size() < 12 + (size_t)NF * (8 + fb)) return 2;
    std::vector<double> ts(NF);
    for (int i = 0; i < NF; i++) memcpy(&ts[i], &raw[12 + (size_t)i * (8 + fb)], 8);
    std::vector<unsigned char> imu_raw;
    if (!skv.count("ImuSamples") || !read_all(skv["ImuSamples"].c_str(), imu_raw) || imu_raw.size() % (7 * 8)) {
        fprintf(stderr, "ImuSamples=<file of float64 rows t, gyro xyz, accel xyz> is required\n");
        return 2;
    }
    const int NS = (int)(imu_raw.size() / (7 * 8));
    std::vector<double> smp(7 * (size_t)NS);
    memcpy(smp.data(), imu_raw.data(), imu_raw.size());

    // Every field must be set: REBVOParameters has no defaults (include/rebvo/rebvo.h:64-235).  Values as
    // oracle/ref_driver.cpp, with ImuMode=1 (the live block of ros/src/rebvo_ros/config/rebvo_EuRoC.yaml).
    REBVOParameters p;
    p.CameraType = 3;
    p.VideoNetHost = "127.0.0.1";
    p.VideoNetPort = 2708;
    p.VideoNetEnabled = false;
    p.BlockingUDP = false;
    p.VideoSave = 0;
    p.VideoSaveFile = "/tmp/ref_video.bin";
    p.VideoSaveBuffersize = 0;
    p.encoder_type = 0;
    p.encoder_dev = "";
    p.EdgeMapDelay = 0;
    p.SaveLog = false;
    p.LogFile = "/tmp/ref_log.m";
    p.TrayFile = "/tmp/ref_tray.txt";
    p.TrackKeyFrames = false;
    p.KFSavePercent = 0.7;
    p.StereoAvaiable = false;
    p.DataSetFile = p.DataSetDir = p.DataSetFileStereo = p.DataSetDirStereo = "";
    p.CamTimeScale = 1;
    p.ImageSize = {(uint)W, (uint)H};
    p.z_f_x = get("ZfX", 458.654);
    p.z_f_y = get("ZfY", 457.296);
    p.pp_x = get("PPx", 367.215);
    p.pp_y = get("PPy", 248.375);
    p.kc = {0, 0, 0, 0, 0};
    p.config_fps = get("FPS", 20);
    p.soft_fps = 1e6;
    p.useUndistort = false;
    p.rotatedCam = false;
    p.CameraDevice = "";
    p.z_f_x_stereo = p.z_f_x;
    p.z_f_y_stereo = p.z_f_y;
    p.pp_x_stereo = p.pp_x;
    p.pp_y_stereo = p.pp_y;
    p.kc_stereo = {0, 0, 0, 0, 0};
    p.SimFile = "";
    p.sim_save_nframes = 0;
    p.simu_time_on = 0;
    p.simu_time_step = 0;
    p.simu_time_sweep = 0;
    p.simu_time_start = 0;
    p.ImuMode = 1;
    p.ImuFile = "";
    p.SE3File = "";
    p.UseCamIMUSE3File = false;
    p.ImuTimeScale = 1;
    p.InitBias = get("InitBias", 0) != 0;
    p.InitBiasFrameNum = (int)get("InitBiasFrameNum", 10);
    p.BiasInitGuess = TooN::Zeros;
    p.GiroMeasStdDev = 1.6968e-4;
    p.GiroBiasStdDev = 1.9393e-5;
    p.AcelMeasStdDev = 2e-3;
    p.g_module = 9.8;
    p.g_module_uncer = 100e3;
    p.g_uncert = 2e-3;
    p.VBiasStdDev = 1e-7;
    p.ScaleStdDevMult = 1e-2;
    p.ScaleStdDevMax = 1e-4;
    p.ScaleStdDevInit = 1.2e-3;
    p.SampleTime = get("SampleTime", 0.005);
    p.CircBufferSize = (int)get("CircBufferSize", 1000);
    p.TimeDesinc = get("TimeDesinc", 0);
    p.cpuSetAffinity = 0;
    p.cpu0 = 0;
    p.cpu1 = 1;
    p.cpu2 = 2;
    p.Sigma0 = get("Sigma0", 3.56359);
    p.KSigma = get("KSigma", 1.2599);
    p.DetectorPlaneFitSize = (int)get("DetectorPlaneFitSize", 2);
    p.DetectorPosNegThresh = get("DetectorPosNegThresh", 0.4);
    p.DetectorDoGThresh = get("DetectorDoGThresh", 0.095259868922420);
    p.ReferencePoints = (int)get("ReferencePoints", 15000);
    p.TrackPoints = (int)get("TrackPoints", 12000);
    p.MaxPoints = (int)get("MaxPoints", 40000);
    p.DetectorThresh = get("DetectorThresh", 0.01);
    p.DetectorAutoGain = get("DetectorAutoGain", 5e-7);
    p.DetectorMaxThresh = get("DetectorMaxThresh", 0.5);
    p.DetectorMinThresh = get("DetectorMinThresh", 0.005);
    p.MatchThreshold = (int)get("GlobalMatchThreshold", 500);
    p.SearchRange = get("SearchRange", 40);
    p.QCutOffNumBins = get("QCutOffNumBins", 100);
    p.QCutOffQuantile = get("QCutOffQuantile", 0.9);
    p.TrackerIterNum = (int)get("TrackerIterNum", 5);
    p.TrackerInitIterNum = (int)get("TrackerInitIterNum", 2);
    p.TrackerInitType = (int)get("TrackerInitType", 2);
    p.TrackerMatchThresh = get("TrackerMatchThresh", 0.5);
    p.LocationUncertaintyMatch = get("LocationUncertaintyMatch", 2);
    p.MatchThreshModule = get("MatchThreshModule", 1);
    p.MatchThreshAngle = get("MatchThreshAngle", 45);
    p.ReweigthDistance = get("ReweigthDistance", 2);
    p.MatchNumThresh = (uint)get("MatchNumThresh", 0);
    p.RegularizeThresh = get("RegularizeThresh", 0.5);
    p.ReshapeQAbsolute = get("ReshapeQAbsolute", 1e-4);
    p.ReshapeQRelative = get("ReshapeQRelative", 1.6968e-4);
    p.LocationUncertainty = get("LocationUncertainty", 1);
    p.DoReScaling = get("DoReScaling", 0);

    g_out.reserve(NF + 8);
    REBVO cf(p);
    cf.setOutputCallback(callback);
    if (!cf.Init()) {
        fprintf(stderr, "REBVO init failed\n");
        return 3;
    }
    auto t0 = std::chrono::steady_clock::now();
    int next = 0;   // next sample to push
    for (int i = 0; i < NF && cf.Running(); i++) {
        // the samples up to frame i's time and the first one past it (its window must end at or before a sample)
        const double tf = ts[i] + p.TimeDesinc;
        while (next < NS && (next == 0 || smp[7 * (size_t)(next - 1)] <= tf)) {
            const double *r = &smp[7 * (size_t)next];
            cf.pushIMU(ImuData(r[0], TooN::makeVector(r[1], r[2], r[3]), TooN::makeVector(r[4], r[5], r[6])));
            next++;
        }
        std::shared_ptr<Image<RGB24Pixel>> ptr;
        while (!cf.requestCustomCamBuffer(ptr, ts[i], 0.5) && cf.Running()) {
        }
        memcpy((*ptr).Data(), &raw[12 + (size_t)i * (8 + fb) + 8], fb);
        cf.releaseCustomCamBuffer();
    }
    // the last frame's window may still wait for a sample past it: hand over the rest
    for (; next < NS; next++) {
        const double *r = &smp[7 * (size_t)next];
        cf.pushIMU(ImuData(r[0], TooN::makeVector(r[1], r[2], r[3]), TooN::makeVector(r[4], r[5], r[6])));
    }
    // An edge map reaches the callback only after it has served as old_buf, i.e. NF-2 callbacks.
    auto deadline = std::chrono::steady_clock::now() + std::chrono::seconds(30);
    while (g_ncb < NF - 2 && std::chrono::steady_clock::now() < deadline) usleep(1000);
    const double wall = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    const int ncb = g_ncb;
    cf.CleanUp();

    FILE *fo = fopen(argv[2], "wb");
    if (fo) {
        int n = (int)g_out.size(), sz = (int)sizeof(OutRec);
        fwrite(&n, 4, 1, fo);
        fwrite(&sz, 4, 1, fo);
        fwrite(g_out.data(), sizeof(OutRec), g_out.size(), fo);
        fclose(fo);
    }
    printf("{\"frames_in\": %d, \"callbacks\": %d, \"timed_callbacks\": %d, \"wall_s\": %.6f, \"fps\": %.4f, "
           "\"samples_pushed\": %d}\n",
           NF, ncb, ncb, wall, ncb / wall, next);
    return 0;
}
