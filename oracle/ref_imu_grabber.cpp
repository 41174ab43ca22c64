// TEST INFRASTRUCTURE ONLY: the reference's live ImuGrabber (src/UtilLib/imugrabber.cpp, unmodified) behind a C interface,
// for tests/test_cpu_imu_live.py: ImuGrabber(list_size, tsamp), PushData, GrabAndIntegrate.
#include <stdexcept>
#include <vector>

#include "UtilLib/imugrabber.h"

using namespace rebvo;

extern "C" {
void *ref_imu_grabber_new(int list_size, double tsample) { return new ImuGrabber(list_size, tsample); }
void ref_imu_grabber_free(void *g) { delete (ImuGrabber *)g; }
// PushData of n rows {t, gyro xyz, accel xyz} one by one: the number stored before the first overflow_error
int ref_imu_grabber_push(void *g, const double *rows, int n) {
    for (int i = 0; i < n; i++) {
        const double *r = rows + 7 * i;
        try {
            ((ImuGrabber *)g)->PushData(ImuData(r[0], TooN::makeVector(r[1], r[2], r[3]), TooN::makeVector(r[4], r[5], r[6])));
        } catch (const std::overflow_error &) {
            return i;
        }
    }
    return n;
}
// GrabAndIntegrate(tstart, tend): out = {n, dt, Rot (row-major), giro, acel, cacel, dgiro} (23 doubles)
void ref_imu_grabber_grab(void *g, double tstart, double tend, double *out) {
    const IntegratedImuData d = ((ImuGrabber *)g)->GrabAndIntegrate(tstart, tend);
    out[0] = d.n;
    out[1] = d.dt;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) out[2 + i * 3 + j] = d.Rot(i, j);
    for (int k = 0; k < 3; k++) {
        out[11 + k] = d.giro[k];
        out[14 + k] = d.acel[k];
        out[17 + k] = d.cacel[k];
        out[20 + k] = d.dgiro[k];
    }
}
}
