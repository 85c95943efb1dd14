// tests/host/system_cpu_preset.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libalva_b200.so).
// The CPU oracle build of the System state machine with the reference's preset switch (state.hpp:9-17): the CLAHE backend of
// system_cpu_clahe.cpp with the grid cell size of the preset in the detector (map_manager.cpp:213) and in the local-map
// matcher's frame grid (frame.cpp:14-15, 308-341).  Under DEFAULT it computes what system_cpu_backend.cpp computes.
// C entry points: cpu_preset_system_*.
#include "system_cpu_clahe.cpp"

// orc_match_to_map_cell: oracle/match_dist_oracle.c's procedure on a grid of orc_match_cell-px cells (tests/preset_util.py
// builds it; with cell 40 and no distortion it is orc_match_to_map)
extern "C" int orc_match_cell;
extern "C" int orc_match_to_map_cell(int w, int h, double fx, double fy, double cx, double cy, const double* Twc_cur, int n_kp,
                                     const int32_t* kp_id, const float* kp_px, int nkp3d, int n_kf, const int32_t* kf_id,
                                     const double* kf_Twc, int n_mp, const int32_t* mp_id, const double* mp_wpt, const uint8_t* mp_is3d,
                                     const int32_t* obs_start, const int32_t* obs_kf, const float* obs_px, const int32_t* desc_start,
                                     const int32_t* desc_kf, const uint8_t* desc, int n_local, const int32_t* local_ids,
                                     float max_proj_err, float dist_ratio, int32_t* match_kp, int32_t* match_mp, const double* dist4);

struct CpuPresetBackend : CpuClaheBackend {
    int cell = 40;   // State::frameMaxCellSize_

    int detect(const float* cpts, int ncur, std::vector<float>& fresh) {
        const int roi[4] = {20, 20, w - 40, h - 40};
        const int cap = 2 * (w / cell) * (h / cell) + 64;
        fresh.assign((size_t)cap * 2, 0.f);
        const int n = orc_detect_points(img[cur][0].data(), w, h, cell, cpts, ncur, roi, &quality, fresh.data(), nullptr, cap);
        fresh.resize((size_t)2 * (n < cap ? n : cap));
        return 0;
    }
    int match_to_map(const alva_sys::MatchProblem& m, std::vector<int>& kp_match) {
        const int n_kp = (int)m.kp_id.size(), n_mp = (int)m.mp_id.size();
        std::vector<int32_t> obs_kf(m.obs_kfid.size()), local_ids(m.local_mp.size()), mk(n_kp + 1), mm(n_kp + 1);
        for (size_t o = 0; o < obs_kf.size(); o++) { int ki = 0; while (m.kf_id[ki] != m.obs_kfid[o]) ki++; obs_kf[o] = ki; }
        for (size_t i = 0; i < local_ids.size(); i++) local_ids[i] = m.mp_id[m.local_mp[i]];
        orc_match_cell = cell;
        const int n = orc_match_to_map_cell(w, h, fx, fy, cx, cy, m.Twc_cur, n_kp, m.kp_id.data(), m.kp_px.data(), m.nkp3d, (int)m.kf_id.size(),
                                            m.kf_id.data(), m.kf_Twc.data(), n_mp, m.mp_id.data(), m.mp_wpt.data(), m.mp_is3d.data(),
                                            m.obs_start.data(), obs_kf.data(), m.obs_px.data(), m.desc_start.data(), m.desc_kfid.data(),
                                            m.desc.data(), (int)local_ids.size(), local_ids.data(), 2.0f, 0.2f, mk.data(), mm.data(), nullptr);
        for (int i = 0; i < n; i++) {
            int ki = 0, mi = 0;
            while (m.kp_id[ki] != mk[i]) ki++;
            while (m.mp_id[mi] != mm[i]) mi++;
            kp_match[ki] = mi;
        }
        return 0;
    }
};

struct CpuPresetSystem {
    CpuPresetBackend be;
    alva_sys::SystemCore<CpuPresetBackend> core;
    CpuPresetSystem() : core(be) {}
};

extern "C" {
void* cpu_preset_system_create(int w, int h, double fx, double fy, double cx, double cy) {
    CpuPresetSystem* s = new CpuPresetSystem();
    s->be.init(w, h);
    s->be.fx = fx; s->be.fy = fy; s->be.cx = cx; s->be.cy = cy;
    s->core.configure(w, h, fx, fy, cx, cy);
    return s;
}
// State::claheEnabled_ / claheContrastLimit_ / claheTileSize_ with VisualFrontend's grid (visual_frontend.cpp:16-18); -1 = empty grid
int cpu_preset_system_set_clahe(void* p, int enabled, double clip_limit, int tile_size) {
    CpuPresetSystem* s = (CpuPresetSystem*)p;
    const int tx = tile_size > 0 ? s->be.w / tile_size : 0, ty = tile_size > 0 ? s->be.h / tile_size : 0;
    if (tx < 1 || ty < 1) return -1;
    s->be.clahe = enabled != 0; s->be.clip = (float)clip_limit; s->be.tx = tx; s->be.ty = ty;
    return 0;
}
// the table of alva_system_set_preset (include/alva_b200.h): 0 DEFAULT, 1 FAST, 2 AVERAGE, 3 ACCURATE; -1 = unknown
int cpu_preset_system_set_preset(void* p, int preset) {
    static const int cell[4] = {40, 50, 45, 35}, p3p[4] = {1, 1, 0, 0}, clahe[4] = {0, 0, 0, 1};
    static const float ratio[4] = {0.95f, 0.9f, 0.9f, 0.95f};
    if (preset < 0 || preset > 3) return -1;
    CpuPresetSystem* s = (CpuPresetSystem*)p;
    s->be.cell = cell[preset];
    s->core.setPreset(cell[preset], ratio[preset], p3p[preset] != 0);
    return cpu_preset_system_set_clahe(p, clahe[preset], 3.0, 50);
}
void cpu_preset_system_set_essential_hook(void* p, void* fn) {
    ((CpuPresetSystem*)p)->be.essential_hook = (int (*)(const double*, const double*, int, int, float, int, float, float, double*, uint8_t*))fn;
}
void cpu_preset_system_destroy(void* p) { delete (CpuPresetSystem*)p; }
void cpu_preset_system_reset(void* p) { ((CpuPresetSystem*)p)->core.reset(); }
int cpu_preset_system_process(void* p, const uint8_t* rgba, double t_ms, double* Twc7) {
    CpuPresetSystem* s = (CpuPresetSystem*)p;
    const int st = s->core.process(rgba, t_ms);
    s->core.cur.Twc.to7(Twc7);
    return st;
}
int cpu_preset_system_keypoints(void* p, int32_t* ids, float* px, uint8_t* is3d, double* wpt, int cap) {
    CpuPresetSystem* s = (CpuPresetSystem*)p;
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
int cpu_preset_system_info(void* p, int32_t* out8) {
    CpuPresetSystem* s = (CpuPresetSystem*)p;
    out8[0] = s->core.cur.id; out8[1] = s->core.cur.kfid; out8[2] = s->core.cur.n; out8[3] = s->core.cur.n3d;
    out8[4] = s->core.ready_for_init; out8[5] = s->core.n_kf; out8[6] = s->core.cur.nocc; out8[7] = s->core.n_mp_ids;
    return 0;
}
// {frames posed by PnP from the prior, p3pReq_ fallbacks, local BA solves, solves under the 21-free-pose limit, max_kps, cell}
int cpu_preset_system_counters(void* p, int32_t* out6) {
    CpuPresetSystem* s = (CpuPresetSystem*)p;
    out6[0] = s->core.n_pnp_prior; out6[1] = s->core.n_p3p_fallback; out6[2] = s->core.n_local_ba; out6[3] = s->core.n_free_pose_clamp;
    out6[4] = s->core.max_kps; out6[5] = s->core.cell;
    return 0;
}
}
