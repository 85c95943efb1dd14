// tests/host/system_cpu_map.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libalva_b200.so).
// The CPU oracle build of the System state machine with relocalisation (system_cpu_reloc.cpp) plus the map blob
// (alva_system_save_map / alva_system_load_map) and the fisheye switch; with the fisheye lens on, the local-map matcher is
// orc_match_to_map_fisheye (built by tests/fisheye_util.py).  C entry points: cpu_map_system_*, next to the cpu_reloc_system_*
// ones, on the same handles.
#include "system_cpu_reloc.cpp"

extern "C" int orc_match_to_map_fisheye(int w, int h, double fx, double fy, double cx, double cy, const double* Twc_cur, int n_kp,
                                        const int32_t* kp_id, const float* kp_px, int nkp3d, int n_kf, const int32_t* kf_id,
                                        const double* kf_Twc, int n_mp, const int32_t* mp_id, const double* mp_wpt, const uint8_t* mp_is3d,
                                        const int32_t* obs_start, const int32_t* obs_kf, const float* obs_px, const int32_t* desc_start,
                                        const int32_t* desc_kf, const uint8_t* desc, int n_local, const int32_t* local_ids,
                                        float max_proj_err, float dist_ratio, int32_t* match_kp, int32_t* match_mp, const double* k4);

struct CpuMapBackend : CpuRelocBackend {
    int match_to_map(const alva_sys::MatchProblem& m, std::vector<int>& kp_match) {
        if (!m.fisheye) return CpuRelocBackend::match_to_map(m, kp_match);
        const int n_kp = (int)m.kp_id.size(), n_mp = (int)m.mp_id.size();
        std::vector<int32_t> obs_kf(m.obs_kfid.size()), local_ids(m.local_mp.size()), mk(n_kp + 1), mm(n_kp + 1);
        for (size_t o = 0; o < obs_kf.size(); o++) { int ki = 0; while (m.kf_id[ki] != m.obs_kfid[o]) ki++; obs_kf[o] = ki; }
        for (size_t i = 0; i < local_ids.size(); i++) local_ids[i] = m.mp_id[m.local_mp[i]];
        const int n = orc_match_to_map_fisheye(w, h, fx, fy, cx, cy, m.Twc_cur, n_kp, m.kp_id.data(), m.kp_px.data(), m.nkp3d,
                                               (int)m.kf_id.size(), m.kf_id.data(), m.kf_Twc.data(), n_mp, m.mp_id.data(), m.mp_wpt.data(),
                                               m.mp_is3d.data(), m.obs_start.data(), obs_kf.data(), m.obs_px.data(), m.desc_start.data(),
                                               m.desc_kfid.data(), m.desc.data(), (int)local_ids.size(), local_ids.data(), 2.0f, 0.2f,
                                               mk.data(), mm.data(), m.dist);
        for (int i = 0; i < n; i++) {
            int ki = 0, mi = 0;
            while (m.kp_id[ki] != mk[i]) ki++;
            while (m.mp_id[mi] != mm[i]) mi++;
            kp_match[ki] = mi;
        }
        return 0;
    }
};

struct CpuMapSystem {
    CpuMapBackend be;
    alva_sys::SystemCore<CpuMapBackend> core;
    CpuMapSystem() : core(be) {}
};

extern "C" {
void* cpu_map_system_create(int w, int h, double fx, double fy, double cx, double cy) {
    CpuMapSystem* s = new CpuMapSystem();
    s->be.init(w, h);
    s->be.fx = fx; s->be.fy = fy; s->be.cx = cx; s->be.cy = cy;
    s->core.configure(w, h, fx, fy, cx, cy);
    return s;
}
void cpu_map_system_destroy(void* p) { delete (CpuMapSystem*)p; }
void cpu_map_system_reset(void* p) { ((CpuMapSystem*)p)->core.reset(); }
int cpu_map_system_set_relocalisation(void* p, int max_lost_frames) {
    if (max_lost_frames < 0) return -1;
    ((CpuMapSystem*)p)->core.setRelocalisation(max_lost_frames);
    return 0;
}
// the table of alva_system_set_preset (include/alva_b200.h): 0 DEFAULT, 1 FAST, 2 AVERAGE, 3 ACCURATE; -1 = unknown
int cpu_map_system_set_preset(void* p, int preset) {
    static const int cell[4] = {40, 50, 45, 35}, p3p[4] = {1, 1, 0, 0}, clahe[4] = {0, 0, 0, 1};
    static const float ratio[4] = {0.95f, 0.9f, 0.9f, 0.95f};
    if (preset < 0 || preset > 3) return -1;
    CpuMapSystem* s = (CpuMapSystem*)p;
    s->be.cell = cell[preset];
    s->core.setPreset(cell[preset], ratio[preset], p3p[preset] != 0);
    s->be.clahe = clahe[preset] != 0; s->be.clip = 3.f; s->be.tx = s->be.w / 50; s->be.ty = s->be.h / 50;
    return 0;
}
void cpu_map_system_set_distortion(void* p, double k1, double k2, double p1, double p2) {
    const double d[4] = {k1, k2, p1, p2};
    ((CpuMapSystem*)p)->core.setDistortion(d);
}
void cpu_map_system_set_fisheye(void* p, int enabled, double k1, double k2, double k3, double k4) {
    const double k[4] = {k1, k2, k3, k4};
    ((CpuMapSystem*)p)->core.setFisheye(enabled != 0, k);
}
int cpu_map_system_process(void* p, const uint8_t* rgba, double t_ms, double* Twc7) {
    CpuMapSystem* s = (CpuMapSystem*)p;
    const int st = s->core.process(rgba, t_ms);
    s->core.cur.Twc.to7(Twc7);
    return st;
}
int cpu_map_system_keypoints(void* p, int32_t* ids, float* px, uint8_t* is3d, int cap) {
    CpuMapSystem* s = (CpuMapSystem*)p;
    int n = 0;
    for (auto& kv : s->core.cur.kps) {
        if (n < cap) { ids[n] = kv.second.id; px[2 * n] = kv.second.px; px[2 * n + 1] = kv.second.py; is3d[n] = kv.second.is3d; }
        n++;
    }
    return n;
}
// {frame id, keyframe id, #keypoints, #3-D keypoints, initialised, #keyframes, #occupied cells, #map point ids}
int cpu_map_system_info(void* p, int32_t* out8) {
    CpuMapSystem* s = (CpuMapSystem*)p;
    out8[0] = s->core.cur.id; out8[1] = s->core.cur.kfid; out8[2] = s->core.cur.n; out8[3] = s->core.cur.n3d;
    out8[4] = s->core.ready_for_init; out8[5] = s->core.n_kf; out8[6] = s->core.cur.nocc; out8[7] = s->core.n_mp_ids;
    return 0;
}
// {n_kf_ids, n_mp_ids, lost now, lost frames, map points in the relocalisation table, its version, keyframes, map points}
int cpu_map_system_counters(void* p, int32_t* out8) {
    CpuMapSystem* s = (CpuMapSystem*)p;
    out8[0] = s->core.n_kf_ids; out8[1] = s->core.n_mp_ids; out8[2] = s->core.lost ? 1 : 0; out8[3] = s->core.lost_frames;
    out8[4] = (int32_t)s->core.reloc_table.mp_id.size(); out8[5] = (int32_t)s->core.reloc_table.version;
    out8[6] = (int32_t)s->core.keyframes.size(); out8[7] = (int32_t)s->core.mappoints.size();
    return 0;
}
// the contract of alva_system_save_map: buf = NULL queries the size; a short buffer gives -3 (ALVA_E_CAPACITY) with *bytes set
int cpu_map_system_save(void* p, uint8_t* buf, size_t cap, size_t* bytes) {
    CpuMapSystem* s = (CpuMapSystem*)p;
    std::vector<uint8_t> blob;
    const int e = s->core.saveMap(blob);
    if (e) return e;
    *bytes = blob.size();
    if (!buf) return 0;
    if (cap < blob.size()) return -3;
    memcpy(buf, blob.data(), blob.size());
    return 0;
}
int cpu_map_system_load(void* p, const uint8_t* buf, size_t bytes) { return ((CpuMapSystem*)p)->core.loadMap(buf, bytes); }
const char* cpu_map_system_error(void* p) { return ((CpuMapSystem*)p)->core.map_error; }
}
