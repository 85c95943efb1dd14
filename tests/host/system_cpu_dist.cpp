// tests/host/system_cpu_dist.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libalva_b200.so).
// The CPU oracle build of the System state machine (system_cpu_backend.cpp) with the lens-distortion switch: the state
// machine applies the model itself through Camera (alvaar_b200/csrc/camera_model.h, host side) -- this backend has no unpx()
// hook -- and the local-map matcher is orc_match_to_map_dist.  With zero coefficients it is exactly the backend of
// system_cpu_backend.cpp.  C entry points: cpu_dist_system_*, one per cpu_system_* of that file, plus cpu_system_set_distortion,
// and the header's host side on point arrays (cpu_cam_undistort_points / cpu_cam_project_points).
#include "system_cpu_backend.cpp"

// orc_match_to_map_dist: oracle/match_dist_oracle.c (linked from tests/_build/libcamera_oracle.so, tests/camera_util.py)
extern "C" int orc_match_to_map_dist(int w, int h, double fx, double fy, double cx, double cy, const double* Twc_cur, int n_kp,
                                     const int32_t* kp_id, const float* kp_px, int nkp3d, int n_kf, const int32_t* kf_id,
                                     const double* kf_Twc, int n_mp, const int32_t* mp_id, const double* mp_wpt, const uint8_t* mp_is3d,
                                     const int32_t* obs_start, const int32_t* obs_kf, const float* obs_px, const int32_t* desc_start,
                                     const int32_t* desc_kf, const uint8_t* desc, int n_local, const int32_t* local_ids,
                                     float max_proj_err, float dist_ratio, int32_t* match_kp, int32_t* match_mp, const double* dist4);

struct CpuDistBackend : CpuBackend {
    int match_to_map(const alva_sys::MatchProblem& m, std::vector<int>& kp_match) {
        const int n_kp = (int)m.kp_id.size(), n_mp = (int)m.mp_id.size();
        std::vector<int32_t> obs_kf(m.obs_kfid.size()), local_ids(m.local_mp.size()), mk(n_kp + 1), mm(n_kp + 1);
        for (size_t o = 0; o < obs_kf.size(); o++) { int ki = 0; while (m.kf_id[ki] != m.obs_kfid[o]) ki++; obs_kf[o] = ki; }
        for (size_t i = 0; i < local_ids.size(); i++) local_ids[i] = m.mp_id[m.local_mp[i]];
        const int n = orc_match_to_map_dist(w, h, fx, fy, cx, cy, m.Twc_cur, n_kp, m.kp_id.data(), m.kp_px.data(), m.nkp3d, (int)m.kf_id.size(),
                                            m.kf_id.data(), m.kf_Twc.data(), n_mp, m.mp_id.data(), m.mp_wpt.data(), m.mp_is3d.data(),
                                            m.obs_start.data(), obs_kf.data(), m.obs_px.data(), m.desc_start.data(), m.desc_kfid.data(),
                                            m.desc.data(), (int)local_ids.size(), local_ids.data(), 2.0f, 0.2f, mk.data(), mm.data(),
                                            m.has_dist ? m.dist : nullptr);
        for (int i = 0; i < n; i++) {
            int ki = 0, mi = 0;
            while (m.kp_id[ki] != mk[i]) ki++;
            while (m.mp_id[mi] != mm[i]) mi++;
            kp_match[ki] = mi;
        }
        return 0;
    }
};

struct CpuDistSystem {
    CpuDistBackend be;
    alva_sys::SystemCore<CpuDistBackend> core;
    CpuDistSystem() : core(be) {}
};

extern "C" {
void* cpu_dist_system_create(int w, int h, double fx, double fy, double cx, double cy) {
    CpuDistSystem* s = new CpuDistSystem();
    s->be.init(w, h);
    s->be.fx = fx; s->be.fy = fy; s->be.cx = cx; s->be.cy = cy;
    s->core.configure(w, h, fx, fy, cx, cy);
    return s;
}
// System::setDistortion: the coefficients of every later frame; resets the tracker and the map
void cpu_system_set_distortion(void* p, double k1, double k2, double p1, double p2) {
    const double d[4] = {k1, k2, p1, p2};
    ((CpuDistSystem*)p)->core.setDistortion(d);
}
void cpu_dist_system_set_essential_hook(void* p, void* fn) {
    ((CpuDistSystem*)p)->be.essential_hook = (int (*)(const double*, const double*, int, int, float, int, float, float, double*, uint8_t*))fn;
}
void cpu_dist_system_destroy(void* p) { delete (CpuDistSystem*)p; }
int cpu_dist_system_process(void* p, const uint8_t* rgba, double t_ms, double* Twc7) {
    CpuDistSystem* s = (CpuDistSystem*)p;
    const int st = s->core.process(rgba, t_ms);
    s->core.cur.Twc.to7(Twc7);
    return st;
}
int cpu_dist_system_keypoints(void* p, int32_t* ids, float* px, uint8_t* is3d, double* wpt, int cap) {
    CpuDistSystem* s = (CpuDistSystem*)p;
    int n = 0;
    for (auto& kv : s->core.cur.kps) {
        if (n < cap) {
            ids[n] = kv.second.id; px[2 * n] = kv.second.px; px[2 * n + 1] = kv.second.py; is3d[n] = kv.second.is3d;
            auto mp = s->core.mappoints.find(kv.second.id);
            for (int k = 0; k < 3; k++) wpt[3 * n + k] = (mp != s->core.mappoints.end() && mp->second.is3d) ? mp->second.p[k] : 0.0;
        }
        n++;
    }
    return n;
}
// System::getFramePoints: truncated unpx of the 2-D keypoints in the frame's order
int cpu_dist_system_frame_points(void* p, int32_t* xy, int cap) {
    CpuDistSystem* s = (CpuDistSystem*)p;
    int n = 0;
    for (auto& kv : s->core.cur.kps) {
        if (kv.second.is3d) continue;
        if (n < cap) { xy[2 * n] = (int)kv.second.ux; xy[2 * n + 1] = (int)kv.second.uy; }
        n++;
    }
    return n;
}
int cpu_dist_system_info(void* p, int32_t* out8) {
    CpuDistSystem* s = (CpuDistSystem*)p;
    out8[0] = s->core.cur.id; out8[1] = s->core.cur.kfid; out8[2] = s->core.cur.n; out8[3] = s->core.cur.n3d;
    out8[4] = s->core.ready_for_init; out8[5] = s->core.n_kf; out8[6] = s->core.cur.nocc; out8[7] = s->core.n_mp_ids;
    return 0;
}
// the state machine's Camera on point arrays: with all-zero D4 its pinhole forms, else camera_model.h
void cpu_cam_undistort_points(const float* px, int n, const double* K4, const double* D4, float* unpx) {
    alva_sys::Camera c;
    c.fx = K4[0]; c.fy = K4[1]; c.cx = K4[2]; c.cy = K4[3];
    c.prepare();
    c.setDistortion(D4);
    for (int i = 0; i < n; i++) c.undistort(px[2 * i], px[2 * i + 1], unpx[2 * i], unpx[2 * i + 1]);
}
void cpu_cam_project_points(const double* Xc, int n, const double* K4, const double* D4, float* uv) {
    alva_sys::Camera c;
    c.fx = K4[0]; c.fy = K4[1]; c.cx = K4[2]; c.cy = K4[3];
    c.prepare();
    c.setDistortion(D4);
    for (int i = 0; i < n; i++) c.projCamToImageDist(Xc + 3 * i, uv[2 * i], uv[2 * i + 1]);
}
// camera_model.h directly: the radial-tangential path whatever the coefficients (zero included)
void cpu_radtan_undistort_points(const float* px, int n, const double* K4, const double* D4, float* unpx) {
    for (int i = 0; i < n; i++) alva_cam::undistort_point(K4, D4, px[2 * i], px[2 * i + 1], unpx + 2 * i);
}
void cpu_radtan_project_points(const double* Xc, int n, const double* K4, const double* D4, float* uv) {
    for (int i = 0; i < n; i++) alva_cam::project_dist(K4, D4, Xc + 3 * i, uv + 2 * i);
}
}
