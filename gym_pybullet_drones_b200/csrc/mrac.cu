// mrac.cu -- qs_mrac_control / qs_mrac_control_state: MRAC.computeControl for n drones, one thread each (include/quadsim.h).
// The per-drone math is mrac_core.cuh; rollout_ctrl.cu runs the same function inside the control-env rollout.
#include "qs_common.cuh"
#include "mrac_core.cuh"

namespace qsi {
namespace {

constexpr int kMracTPB = 128;

struct MracArgs {
    QsMracParams M;
    double* state;
    double dt;
    const double *pos, *quat, *vel, *angv;        // qs_mrac_control; NULL for qs_mrac_control_state
    const double* planes;                         // qs_mrac_control_state
    const double *tpos, *trpy, *tvel, *trr;
    long long n;
    double* rpm_out;
    float *pos_e_out, *rpy_e_out;
    double max_rpm;                               // qs_mrac_control_state: clip to [0, max_rpm]; < 0: no clip
    int init;
};

__device__ __forceinline__ void ld3(const double* p, long long i, double v[3]) {
    if (p) { v[0] = p[3 * i]; v[1] = p[3 * i + 1]; v[2] = p[3 * i + 2]; } else { v[0] = v[1] = v[2] = 0.0; }
}

__global__ void __launch_bounds__(kMracTPB) mrac_kernel(const __grid_constant__ MracArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long N = a.n;
    if (i >= N) return;
    double pos[3], quat[4], vel[3], av[3], r[12];
    if (a.planes) {
        qs::Drone d;
        load_drone(a.planes, N, i, d);
        pos[0] = d.px; pos[1] = d.py; pos[2] = d.pz;
        quat[0] = d.qx; quat[1] = d.qy; quat[2] = d.qz; quat[3] = d.qw;
        vel[0] = d.vx; vel[1] = d.vy; vel[2] = d.vz;
        qs::mrac_ang_v(d, av);
    } else {
        ld3(a.pos, i, pos); ld3(a.vel, i, vel); ld3(a.angv, i, av);
        quat[0] = a.quat[4 * i]; quat[1] = a.quat[4 * i + 1]; quat[2] = a.quat[4 * i + 2]; quat[3] = a.quat[4 * i + 3];
    }
    ld3(a.tpos, i, r); ld3(a.trpy, i, r + 3); ld3(a.tvel, i, r + 6); ld3(a.trr, i, r + 9);
    double rpm[4], pe[3], ye[3];
    const qs::MracState S = {a.state + i, N};
    qs::mrac_control(a.M, S, a.init != 0, a.dt, pos, quat, vel, av, r, rpm, pe, ye);
    if (a.max_rpm >= 0.0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) rpm[j] = qs::clampd(rpm[j], 0.0, a.max_rpm);             // CtrlAviary.py:140
    }
    st256(a.rpm_out, i, rpm[0], rpm[1], rpm[2], rpm[3]);
    if (a.pos_e_out) { a.pos_e_out[3 * i] = (float)pe[0]; a.pos_e_out[3 * i + 1] = (float)pe[1]; a.pos_e_out[3 * i + 2] = (float)pe[2]; }
    if (a.rpy_e_out) { a.rpy_e_out[3 * i] = (float)ye[0]; a.rpy_e_out[3 * i + 1] = (float)ye[1]; a.rpy_e_out[3 * i + 2] = (float)ye[2]; }
}

int launch_mrac(const MracArgs& a, void* stream, const char* what) {
    mrac_kernel<<<(unsigned)((a.n + kMracTPB - 1) / kMracTPB), kMracTPB, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, what);
}

}  // namespace
}  // namespace qsi

using namespace qsi;

extern "C" {

int qs_sizeof_mrac_params(void) { return (int)sizeof(QsMracParams); }

int qs_mrac_control(const QsMracParams* p, double* mrac_state, int init, double control_timestep,
                    const double* cur_pos, const double* cur_quat, const double* cur_vel, const double* cur_ang_vel,
                    const double* target_pos, const double* target_rpy, const double* target_vel, const double* target_rpy_rates,
                    int n, double* rpm_out, float* pos_e_out, float* rpy_e_out, void* stream) {
    if (!p || !mrac_state || !cur_pos || !cur_quat || !cur_vel || !cur_ang_vel || !target_pos || !rpm_out)
        return fail(QS_ERR_NULL, "qs_mrac_control: NULL argument");
    if (n <= 0) return fail(QS_ERR_SIZE, "qs_mrac_control: n must be > 0");
    if (!(control_timestep > 0.0)) return fail(QS_ERR_SIZE, "qs_mrac_control: control_timestep must be > 0");
    if (!aligned32(rpm_out)) return fail(QS_ERR_ALIGN, "qs_mrac_control: rpm_out must be 32-byte aligned");
    MracArgs a;
    memset(&a, 0, sizeof(a));
    a.M = *p; a.state = mrac_state; a.dt = control_timestep; a.init = init;
    a.pos = cur_pos; a.quat = cur_quat; a.vel = cur_vel; a.angv = cur_ang_vel;
    a.tpos = target_pos; a.trpy = target_rpy; a.tvel = target_vel; a.trr = target_rpy_rates; a.n = n;
    a.rpm_out = rpm_out; a.pos_e_out = pos_e_out; a.rpy_e_out = rpy_e_out; a.max_rpm = -1.0;
    return launch_mrac(a, stream, "qs_mrac_control launch");
}

int qs_mrac_control_state(const QsMracParams* p, double* mrac_state, int init, double control_timestep, const QsState* st, int n,
                          const double* target_pos, const double* target_rpy, const double* target_vel, const double* target_rpy_rates,
                          double* rpm_out, float* pos_e_out, float* rpy_e_out, void* stream) {
    if (!p || !mrac_state || !st || !st->planes || !target_pos || !rpm_out) return fail(QS_ERR_NULL, "qs_mrac_control_state: NULL argument");
    if (n <= 0) return fail(QS_ERR_SIZE, "qs_mrac_control_state: n must be > 0");
    if (!(control_timestep > 0.0)) return fail(QS_ERR_SIZE, "qs_mrac_control_state: control_timestep must be > 0");
    if (!aligned32(st->planes) || !aligned32(rpm_out)) return fail(QS_ERR_ALIGN, "qs_mrac_control_state: planes / rpm_out must be 32-byte aligned");
    MracArgs a;
    memset(&a, 0, sizeof(a));
    a.M = *p; a.state = mrac_state; a.dt = control_timestep; a.init = init; a.planes = st->planes;
    a.tpos = target_pos; a.trpy = target_rpy; a.tvel = target_vel; a.trr = target_rpy_rates; a.n = n;
    a.rpm_out = rpm_out; a.pos_e_out = pos_e_out; a.rpy_e_out = rpy_e_out; a.max_rpm = p->max_rpm;
    return launch_mrac(a, stream, "qs_mrac_control_state launch");
}

}  // extern "C"
