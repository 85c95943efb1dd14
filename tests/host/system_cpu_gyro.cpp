// tests/host/system_cpu_gyro.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libalva_b200.so).
// The CPU oracle build of the System state machine with relocalisation, the map blob and the localisation-only mode
// (system_cpu_localisation.cpp) plus the gyro mode: Backend::klt_rotated replaces the flagged KLT priors through
// alva_cam::rotate_prior (alvaar_b200/csrc/camera_model.h, host side -- the arithmetic alva_k_rotate_priors runs on the device)
// and then runs orc_fb_klt (oracle/klt_oracle.c) as klt() does.  C entry points: cpu_gyro_system_*, and cpu_gyro_rotate_priors,
// the host build of alva_k_rotate_priors.
#include "system_cpu_localisation.cpp"

struct CpuGyroBackend : CpuLocBackend {
    int klt_rotated(const float* pts, float* priors, int n, int levels, uint8_t* good, const double* bv, const uint8_t* flag,
                    const double* dR9, uint8_t* rotated) {
        const double K4[4] = {fx, fy, cx, cy};
        for (int i = 0; i < n; i++)
            rotated[i] = flag[i] && alva_cam::rotate_prior(lens, K4, coef, w, h, dR9, bv + 3 * (size_t)i, priors + 2 * (size_t)i);
        return klt(pts, priors, n, levels, good);
    }
};

struct CpuGyroSystem {
    CpuGyroBackend be;
    alva_sys::SystemCore<CpuGyroBackend> core;
    CpuGyroSystem() : core(be) {}
};

extern "C" {
void* cpu_gyro_system_create(int w, int h, double fx, double fy, double cx, double cy) {
    CpuGyroSystem* s = new CpuGyroSystem();
    s->be.init(w, h);
    s->be.fx = fx; s->be.fy = fy; s->be.cx = cx; s->be.cy = cy;
    s->core.configure(w, h, fx, fy, cx, cy);
    return s;
}
void cpu_gyro_system_destroy(void* p) { delete (CpuGyroSystem*)p; }
// configure again with the same camera (clears the gyro mode, as alva_system_configure)
void cpu_gyro_system_configure(void* p) {
    CpuGyroSystem* s = (CpuGyroSystem*)p;
    s->core.configure(s->be.w, s->be.h, s->be.fx, s->be.fy, s->be.cx, s->be.cy);
    s->be.lens = 0;
    for (int i = 0; i < 4; i++) s->be.coef[i] = 0.0;
}
void cpu_gyro_system_reset(void* p) { ((CpuGyroSystem*)p)->core.reset(); }
int cpu_gyro_system_set_relocalisation(void* p, int max_lost_frames) {
    if (max_lost_frames < 0) return -1;
    return ((CpuGyroSystem*)p)->core.setRelocalisation(max_lost_frames);
}
void cpu_gyro_system_set_distortion(void* p, double k1, double k2, double p1, double p2) {
    CpuGyroSystem* s = (CpuGyroSystem*)p;
    const double d[4] = {k1, k2, p1, p2};
    s->core.setDistortion(d);
    s->be.lens = s->core.cam.lens;
    for (int i = 0; i < 4; i++) s->be.coef[i] = d[i];
}
void cpu_gyro_system_set_fisheye(void* p, int enabled, double k1, double k2, double k3, double k4) {
    CpuGyroSystem* s = (CpuGyroSystem*)p;
    const double k[4] = {k1, k2, k3, k4};
    s->core.setFisheye(enabled != 0, k);
    s->be.lens = s->core.cam.lens;
    for (int i = 0; i < 4; i++) s->be.coef[i] = enabled ? k[i] : 0.0;
}
// 0, -1 (ALVA_E_INVALID) or -4 (ALVA_E_STATE), as alva_system_set_gyro
int cpu_gyro_system_set_gyro(void* p, int enabled, const double* R_ci9, const double* bias3) {
    if (enabled != 0 && enabled != 1) return -1;
    return ((CpuGyroSystem*)p)->core.setGyro(enabled != 0, R_ci9, bias3);
}
// alva_system_find_camera_pose_gyro: the samples are checked (and kept with the mode on), then the frame is processed; a refusal
// returns -1 and processes no frame
int cpu_gyro_system_process(void* p, const uint8_t* rgba, double t_ms, const double* samples, int n, double* Twc7) {
    CpuGyroSystem* s = (CpuGyroSystem*)p;
    if (int e = s->core.addGyroSamples(samples, n)) return e;
    const int st = s->core.process(rgba, t_ms);
    s->core.cur.Twc.to7(Twc7);
    return st;
}
// alva_system_gyro_stats, plus the samples held
int cpu_gyro_system_stats(void* p, int32_t* out6, double* dR9) {
    const auto& c = ((CpuGyroSystem*)p)->core;
    out6[0] = c.n_gyro_pred; out6[1] = c.n_gyro_fallback; out6[2] = c.n_gyro_carried; out6[3] = c.n_gyro_rot; out6[4] = c.n_gyro_kept;
    out6[5] = (int32_t)c.gyroSamplesHeld();
    memcpy(dR9, c.gyro_dRc, 9 * sizeof(double));
    return 0;
}
int cpu_gyro_system_keypoints(void* p, int32_t* ids, float* px, uint8_t* is3d, int cap) {
    CpuGyroSystem* s = (CpuGyroSystem*)p;
    int n = 0;
    for (auto& kv : s->core.cur.kps) {
        if (n < cap) { ids[n] = kv.second.id; px[2 * n] = kv.second.px; px[2 * n + 1] = kv.second.py; is3d[n] = kv.second.is3d; }
        n++;
    }
    return n;
}
// {frame id, keyframe id, #keypoints, #3-D keypoints, initialised, #keyframes, #occupied cells, #map point ids}
int cpu_gyro_system_info(void* p, int32_t* out8) {
    CpuGyroSystem* s = (CpuGyroSystem*)p;
    out8[0] = s->core.cur.id; out8[1] = s->core.cur.kfid; out8[2] = s->core.cur.n; out8[3] = s->core.cur.n3d;
    out8[4] = s->core.ready_for_init; out8[5] = s->core.n_kf; out8[6] = s->core.cur.nocc; out8[7] = s->core.n_mp_ids;
    return 0;
}
// {times lost, frames relocalised, lost now}
int cpu_gyro_system_counters(void* p, int32_t* out3) {
    const auto& c = ((CpuGyroSystem*)p)->core;
    out3[0] = c.n_lost; out3[1] = c.n_relocalised; out3[2] = c.lost ? 1 : 0;
    return 0;
}
int cpu_gyro_system_save(void* p, uint8_t* buf, size_t cap, size_t* bytes) {
    std::vector<uint8_t> blob;
    const int e = ((CpuGyroSystem*)p)->core.saveMap(blob);
    if (e) return e;
    *bytes = blob.size();
    if (!buf) return 0;
    if (cap < blob.size()) return -3;
    memcpy(buf, blob.data(), blob.size());
    return 0;
}
const char* cpu_gyro_system_error(void* p) { return ((CpuGyroSystem*)p)->core.map_error; }
// the host build of alva_k_rotate_priors (camera_model.h): flagged priors replaced where valid, rotated [n] set
void cpu_gyro_rotate_priors(const double* bv, const uint8_t* flag, int n, int w, int h, const double* K4, const double* D4, int lens,
                            const double* R9, float* prior, uint8_t* rotated) {
    const double zero[4] = {0, 0, 0, 0};
    for (int i = 0; i < n; i++)
        rotated[i] = flag[i] && alva_cam::rotate_prior(lens, K4, D4 ? D4 : zero, w, h, R9, bv + 3 * (size_t)i, prior + 2 * (size_t)i);
}
}
