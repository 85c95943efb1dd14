// tests/host/system_cpu_lens_full.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libalva_b200.so).
// The CPU oracle build of the System state machine (system_cpu_backend.cpp) with OpenCV's whole distortion vector
// (setDistortionCoeffs): the state machine applies the model itself through Camera (alvaar_b200/csrc/camera_model.h, host side)
// -- this backend has no unpx() hook -- and the local-map matcher of lens 3 is orc_match_to_map_full (oracle/match_dist_oracle.c
// with its projection taken through oracle/camera_full_oracle.c, built by tests/camera_full_util.py).  C entry points:
// cpu_full_system_*.
#include "system_cpu_backend.cpp"

extern "C" int orc_match_to_map_full(int w, int h, double fx, double fy, double cx, double cy, const double* Twc_cur, int n_kp,
                                     const int32_t* kp_id, const float* kp_px, int nkp3d, int n_kf, const int32_t* kf_id,
                                     const double* kf_Twc, int n_mp, const int32_t* mp_id, const double* mp_wpt, const uint8_t* mp_is3d,
                                     const int32_t* obs_start, const int32_t* obs_kf, const float* obs_px, const int32_t* desc_start,
                                     const int32_t* desc_kf, const uint8_t* desc, int n_local, const int32_t* local_ids,
                                     float max_proj_err, float dist_ratio, int32_t* match_kp, int32_t* match_mp, const double* k14);

struct CpuFullBackend : CpuBackend {
    int match_to_map(const alva_sys::MatchProblem& m, std::vector<int>& kp_match) {
        if (!m.full) return CpuBackend::match_to_map(m, kp_match);
        const int n_kp = (int)m.kp_id.size(), n_mp = (int)m.mp_id.size();
        std::vector<int32_t> obs_kf(m.obs_kfid.size()), local_ids(m.local_mp.size()), mk(n_kp + 1), mm(n_kp + 1);
        for (size_t o = 0; o < obs_kf.size(); o++) { int ki = 0; while (m.kf_id[ki] != m.obs_kfid[o]) ki++; obs_kf[o] = ki; }
        for (size_t i = 0; i < local_ids.size(); i++) local_ids[i] = m.mp_id[m.local_mp[i]];
        const int n = orc_match_to_map_full(w, h, fx, fy, cx, cy, m.Twc_cur, n_kp, m.kp_id.data(), m.kp_px.data(), m.nkp3d,
                                            (int)m.kf_id.size(), m.kf_id.data(), m.kf_Twc.data(), n_mp, m.mp_id.data(), m.mp_wpt.data(),
                                            m.mp_is3d.data(), m.obs_start.data(), obs_kf.data(), m.obs_px.data(), m.desc_start.data(),
                                            m.desc_kfid.data(), m.desc.data(), (int)local_ids.size(), local_ids.data(), 2.0f, 0.2f,
                                            mk.data(), mm.data(), m.lf.k);
        for (int i = 0; i < n; i++) {
            int ki = 0, mi = 0;
            while (m.kp_id[ki] != mk[i]) ki++;
            while (m.mp_id[mi] != mm[i]) mi++;
            kp_match[ki] = mi;
        }
        return 0;
    }
};

struct CpuFullSystem {
    CpuFullBackend be;
    alva_sys::SystemCore<CpuFullBackend> core;
    CpuFullSystem() : core(be) {}
};

extern "C" {
void* cpu_full_system_create(int w, int h, double fx, double fy, double cx, double cy) {
    CpuFullSystem* s = new CpuFullSystem();
    s->be.init(w, h);
    s->be.fx = fx; s->be.fy = fy; s->be.cx = cx; s->be.cy = cy;
    s->core.configure(w, h, fx, fy, cx, cy);
    return s;
}
// System::setDistortionCoeffs: the model of every later frame; resets the tracker and the map.  -> the lens chosen, -1 refused
int cpu_full_system_set_coeffs(void* p, const double* coeffs, int n) {
    CpuFullSystem* s = (CpuFullSystem*)p;
    return s->core.setDistortionCoeffs(coeffs, n) ? s->core.cam.lens : -1;
}
void cpu_full_system_destroy(void* p) { delete (CpuFullSystem*)p; }
int cpu_full_system_process(void* p, const uint8_t* rgba, double t_ms, double* Twc7) {
    CpuFullSystem* s = (CpuFullSystem*)p;
    const int st = s->core.process(rgba, t_ms);
    s->core.cur.Twc.to7(Twc7);
    return st;
}
int cpu_full_system_keypoints(void* p, int32_t* ids, float* px, uint8_t* is3d, double* wpt, int cap) {
    CpuFullSystem* s = (CpuFullSystem*)p;
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
int cpu_full_system_frame_points(void* p, int32_t* xy, int cap) {
    CpuFullSystem* s = (CpuFullSystem*)p;
    int n = 0;
    for (auto& kv : s->core.cur.kps) {
        if (kv.second.is3d) continue;
        if (n < cap) { xy[2 * n] = (int)kv.second.ux; xy[2 * n + 1] = (int)kv.second.uy; }
        n++;
    }
    return n;
}
int cpu_full_system_info(void* p, int32_t* out8) {
    CpuFullSystem* s = (CpuFullSystem*)p;
    out8[0] = s->core.cur.id; out8[1] = s->core.cur.kfid; out8[2] = s->core.cur.n; out8[3] = s->core.cur.n3d;
    out8[4] = s->core.ready_for_init; out8[5] = s->core.n_kf; out8[6] = s->core.cur.nocc; out8[7] = s->core.n_mp_ids;
    return 0;
}
int cpu_full_system_lens_drops(void* p) { return ((CpuFullSystem*)p)->core.n_lens_drops; }
int cpu_full_system_local_bas(void* p) { return ((CpuFullSystem*)p)->core.n_local_ba; }
}
