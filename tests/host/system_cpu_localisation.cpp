// tests/host/system_cpu_localisation.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libalva_b200.so).
// The CPU oracle build of the System state machine with relocalisation and the map blob (system_cpu_map.cpp, itself built on
// system_cpu_reloc.cpp) plus the localisation-only mode: Backend::reacquire runs oracle/reacquire_oracle.c, the plain-C
// restatement of alva_k_match_frame_to_map, on the same table the device keeps resident.  C entry points: cpu_loc_system_*.
#include "system_cpu_map.cpp"

extern "C" int orc_match_frame_to_map(int w, int h, int cell, double fx, double fy, double cx, double cy, int lens, const double* coef4,
                                      const double* Twc, int n_mp, const double* wpt, const int32_t* desc_start, const uint8_t* desc,
                                      const uint8_t* skip, int nq, const float* q_px, const uint8_t* q_desc, const uint8_t* q_kept,
                                      float radius, int32_t* q_row, int32_t* q_dist);

struct CpuLocBackend : CpuMapBackend {
    int lens = 0;                       // the lens of alva_k_match_frame_to_map: 0 pinhole, 1 radial-tangential, 2 fisheye
    double coef[4] = {0, 0, 0, 0};
    int reacquire(const alva_sys::RelocTable& T, const uint8_t* skip, const double* Twc7, const float* qpx, const uint8_t* qdesc,
                  const uint8_t* qkept, int nq, float radius, int32_t* row, int32_t* dist) {
        static const uint8_t none[32] = {0};
        const int32_t zero = 0;
        const int n = (int)T.mp_id.size();
        return orc_match_frame_to_map(w, h, cell, fx, fy, cx, cy, lens, coef, Twc7, n, T.wpt.data(), n ? T.desc_start.data() : &zero,
                                      T.desc.empty() ? none : T.desc.data(), skip, nq, qpx, qdesc, qkept, radius, row, dist) < 0 ? -1 : 0;
    }
};

struct CpuLocSystem {
    CpuLocBackend be;
    alva_sys::SystemCore<CpuLocBackend> core;
    CpuLocSystem() : core(be) {}
};

extern "C" {
void* cpu_loc_system_create(int w, int h, double fx, double fy, double cx, double cy) {
    CpuLocSystem* s = new CpuLocSystem();
    s->be.init(w, h);
    s->be.fx = fx; s->be.fy = fy; s->be.cx = cx; s->be.cy = cy;
    s->core.configure(w, h, fx, fy, cx, cy);
    return s;
}
void cpu_loc_system_destroy(void* p) { delete (CpuLocSystem*)p; }
void cpu_loc_system_reset(void* p) { ((CpuLocSystem*)p)->core.reset(); }
// 0, -1 (ALVA_E_INVALID) or -4 (ALVA_E_STATE), as alva_system_set_relocalisation
int cpu_loc_system_set_relocalisation(void* p, int max_lost_frames) {
    if (max_lost_frames < 0) return -1;
    return ((CpuLocSystem*)p)->core.setRelocalisation(max_lost_frames);
}
// 0, -1 or -4, as alva_system_set_localisation_only
int cpu_loc_system_set_localisation_only(void* p, int enabled) {
    if (enabled != 0 && enabled != 1) return -1;
    return ((CpuLocSystem*)p)->core.setLocalisationOnly(enabled != 0);
}
// the table of alva_system_set_preset (include/alva_b200.h): 0 DEFAULT, 1 FAST, 2 AVERAGE, 3 ACCURATE; -1 = unknown
int cpu_loc_system_set_preset(void* p, int preset) {
    static const int cell[4] = {40, 50, 45, 35}, p3p[4] = {1, 1, 0, 0}, clahe[4] = {0, 0, 0, 1};
    static const float ratio[4] = {0.95f, 0.9f, 0.9f, 0.95f};
    if (preset < 0 || preset > 3) return -1;
    CpuLocSystem* s = (CpuLocSystem*)p;
    s->be.cell = cell[preset];
    s->core.setPreset(cell[preset], ratio[preset], p3p[preset] != 0);
    s->be.clahe = clahe[preset] != 0; s->be.clip = 3.f; s->be.tx = s->be.w / 50; s->be.ty = s->be.h / 50;
    return 0;
}
// CLAHE alone (alva_system_set_clahe with the preset table's clip and tile): keeps the map and the mode
void cpu_loc_system_set_clahe(void* p, int enabled) {
    CpuLocSystem* s = (CpuLocSystem*)p;
    s->be.clahe = enabled != 0; s->be.clip = 3.f; s->be.tx = s->be.w / 50; s->be.ty = s->be.h / 50;
}
void cpu_loc_system_set_distortion(void* p, double k1, double k2, double p1, double p2) {
    CpuLocSystem* s = (CpuLocSystem*)p;
    const double d[4] = {k1, k2, p1, p2};
    s->core.setDistortion(d);
    s->be.lens = s->core.cam.lens;
    for (int i = 0; i < 4; i++) s->be.coef[i] = d[i];
}
void cpu_loc_system_set_fisheye(void* p, int enabled, double k1, double k2, double k3, double k4) {
    CpuLocSystem* s = (CpuLocSystem*)p;
    const double k[4] = {k1, k2, k3, k4};
    s->core.setFisheye(enabled != 0, k);
    s->be.lens = s->core.cam.lens;
    for (int i = 0; i < 4; i++) s->be.coef[i] = enabled ? k[i] : 0.0;
}
int cpu_loc_system_process(void* p, const uint8_t* rgba, double t_ms, double* Twc7) {
    CpuLocSystem* s = (CpuLocSystem*)p;
    const int st = s->core.process(rgba, t_ms);
    s->core.cur.Twc.to7(Twc7);
    return st;
}
int cpu_loc_system_keypoints(void* p, int32_t* ids, float* px, uint8_t* is3d, int cap) {
    CpuLocSystem* s = (CpuLocSystem*)p;
    int n = 0;
    for (auto& kv : s->core.cur.kps) {
        if (n < cap) { ids[n] = kv.second.id; px[2 * n] = kv.second.px; px[2 * n + 1] = kv.second.py; is3d[n] = kv.second.is3d; }
        n++;
    }
    return n;
}
// {frame id, keyframe id, #keypoints, #3-D keypoints, initialised, #keyframes, #occupied cells, #map point ids}
int cpu_loc_system_info(void* p, int32_t* out8) {
    CpuLocSystem* s = (CpuLocSystem*)p;
    out8[0] = s->core.cur.id; out8[1] = s->core.cur.kfid; out8[2] = s->core.cur.n; out8[3] = s->core.cur.n3d;
    out8[4] = s->core.ready_for_init; out8[5] = s->core.n_kf; out8[6] = s->core.cur.nocc; out8[7] = s->core.n_mp_ids;
    return 0;
}
// {n_kf_ids, n_mp_ids, lost now, lost frames, map points in the relocalisation table, its version, keyframes, map points,
//  mode on, re-acquisition runs, points it supplied, points of its last run, frames relocalised, times lost}
int cpu_loc_system_counters(void* p, int32_t* out14) {
    CpuLocSystem* s = (CpuLocSystem*)p;
    const auto& c = s->core;
    const int32_t v[14] = {c.n_kf_ids, c.n_mp_ids, c.lost ? 1 : 0, c.lost_frames, (int32_t)c.reloc_table.mp_id.size(), (int32_t)c.reloc_table.version,
                           (int32_t)c.keyframes.size(), (int32_t)c.mappoints.size(), c.frozen ? 1 : 0, c.n_reacq_runs, c.n_reacq_points,
                           c.reacq_last_points, c.n_relocalised, c.n_lost};
    memcpy(out14, v, sizeof v);
    return 0;
}
int cpu_loc_system_save(void* p, uint8_t* buf, size_t cap, size_t* bytes) {
    CpuLocSystem* s = (CpuLocSystem*)p;
    std::vector<uint8_t> blob;
    const int e = s->core.saveMap(blob);
    if (e) return e;
    *bytes = blob.size();
    if (!buf) return 0;
    if (cap < blob.size()) return -3;
    memcpy(buf, blob.data(), blob.size());
    return 0;
}
int cpu_loc_system_load(void* p, const uint8_t* buf, size_t bytes) { return ((CpuLocSystem*)p)->core.loadMap(buf, bytes); }
const char* cpu_loc_system_error(void* p) { return ((CpuLocSystem*)p)->core.map_error; }
}
