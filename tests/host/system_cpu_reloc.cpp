// tests/host/system_cpu_reloc.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libalva_b200.so).
// The CPU oracle build of the System state machine with relocalisation (alva_system_set_relocalisation): the preset backend of
// system_cpu_preset.cpp (cell size, CLAHE) with the lens model in its local-map matcher, a detector pass for lost frames with
// its own adaptive quality, and Backend::relocalise on oracle/reloc_oracle.c -- the grouped 2-NN, the match rules and
// P3P-RANSAC -- followed by the P3P -> PnP hand-over the device does (pnp_from_p3p_kernel) and orc_pnp.
// C entry points: cpu_reloc_system_*.
#include "system_cpu_preset.cpp"

extern "C" {
void orc_hamming_knn2_grouped(const uint8_t* q, int nq, const int32_t* desc_start, int n_grp, const uint8_t* desc, int32_t* out);
int orc_reloc_select(const int32_t* knn, int nq, int n_grp, int max_dist, int32_t* mq, int32_t* mg);
int orc_p3p_ransac(const double* bvs, const double* wpts, int n, int max_iter, float err_px, float fx, float fy, uint32_t seed,
                   double* Twc_out, uint8_t* outlier, double* info);
}

struct CpuRelocBackend : CpuPresetBackend {
    double reloc_quality = 0.001;   // the lost frames' detector quality (the tracker's `quality` is left alone)

    int match_to_map(const alva_sys::MatchProblem& m, std::vector<int>& kp_match) {
        const int n_kp = (int)m.kp_id.size(), n_mp = (int)m.mp_id.size();
        std::vector<int32_t> obs_kf(m.obs_kfid.size()), local_ids(m.local_mp.size()), mk(n_kp + 1), mm(n_kp + 1);
        for (size_t o = 0; o < obs_kf.size(); o++) { int ki = 0; while (m.kf_id[ki] != m.obs_kfid[o]) ki++; obs_kf[o] = ki; }
        for (size_t i = 0; i < local_ids.size(); i++) local_ids[i] = m.mp_id[m.local_mp[i]];
        orc_match_cell = cell;
        const int n = orc_match_to_map_cell(w, h, fx, fy, cx, cy, m.Twc_cur, n_kp, m.kp_id.data(), m.kp_px.data(), m.nkp3d, (int)m.kf_id.size(),
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
    int detect_lost(std::vector<float>& fresh) {
        const int roi[4] = {20, 20, w - 40, h - 40};
        const int cap = 2 * (w / cell) * (h / cell) + 64;
        fresh.assign((size_t)cap * 2, 0.f);
        const int n = orc_detect_points(img[cur][0].data(), w, h, cell, nullptr, 0, roi, &reloc_quality, fresh.data(), nullptr, cap);
        fresh.resize((size_t)2 * (n < cap ? n : cap));
        return 0;
    }
    int relocalise(const alva_sys::RelocTable& T, const uint8_t* qdesc, const double* qbv, const double* quv, int nq, const double* K4,
                   float fxf, float fyf, alva_sys::RelocResult& R) {
        R = alva_sys::RelocResult();
        const int n_grp = (int)T.mp_id.size();
        if (nq == 0 || n_grp == 0) return 0;
        std::vector<int32_t> knn(4 * (size_t)nq), mq(nq), mg(nq);
        orc_hamming_knn2_grouped(qdesc, nq, T.desc_start.data(), n_grp, T.desc.data(), knn.data());
        const int n = orc_reloc_select(knn.data(), nq, n_grp, 51, mq.data(), mg.data());
        R.n_match = n;
        R.mq.assign(mq.begin(), mq.begin() + n);
        R.mg.assign(mg.begin(), mg.begin() + n);
        std::vector<double> bv(3 * (size_t)n + 3), X(3 * (size_t)n + 3);
        for (int i = 0; i < n; i++)
            for (int c = 0; c < 3; c++) { bv[3 * i + c] = qbv[3 * (size_t)mq[i] + c]; X[3 * i + c] = T.wpt[3 * (size_t)mg[i] + c]; }
        R.o1.assign(n, 1);
        R.o2.assign(n, 0);
        double info[3];
        R.ok1 = orc_p3p_ransac(bv.data(), X.data(), n, 512, 3.0f, fxf, fyf, 12345u, R.T12, R.o1.data(), info);
        if (info[1] < 0) return 0;   // no model: the device leaves PnP nothing to start from either (ok2 = 0)
        // the hand-over of pnp_from_p3p_kernel: the RANSAC pose as the start (rotation matrix -> quaternion), its inliers in order
        alva_sys::Se3 T0;
        const double Rm[9] = {R.T12[0], R.T12[1], R.T12[2], R.T12[4], R.T12[5], R.T12[6], R.T12[8], R.T12[9], R.T12[10]};
        T0.setR(Rm);
        T0.t[0] = R.T12[3]; T0.t[1] = R.T12[7]; T0.t[2] = R.T12[11];
        T0.to7(R.pose7);
        std::vector<double> uv2, X2;
        for (int i = 0; i < n; i++) {
            if (R.o1[i]) continue;
            uv2.push_back(quv[2 * (size_t)mq[i]]); uv2.push_back(quv[2 * (size_t)mq[i] + 1]);
            X2.insert(X2.end(), &X[3 * i], &X[3 * i] + 3);
        }
        const int n2 = (int)uv2.size() / 2;
        if (n2 < 1) return 0;
        double summary[12];
        const float chi2 = 5.9915f;
        R.ok2 = orc_pnp(K4, uv2.data(), X2.data(), n2, R.pose7, (double)std::sqrt(chi2), (double)chi2, 5, 1, 1, R.o2.data(), summary);
        return 0;
    }
};

struct CpuRelocSystem {
    CpuRelocBackend be;
    alva_sys::SystemCore<CpuRelocBackend> core;
    CpuRelocSystem() : core(be) {}
};

extern "C" {
void* cpu_reloc_system_create(int w, int h, double fx, double fy, double cx, double cy) {
    CpuRelocSystem* s = new CpuRelocSystem();
    s->be.init(w, h);
    s->be.fx = fx; s->be.fy = fy; s->be.cx = cx; s->be.cy = cy;
    s->core.configure(w, h, fx, fy, cx, cy);
    return s;
}
void cpu_reloc_system_destroy(void* p) { delete (CpuRelocSystem*)p; }
void cpu_reloc_system_reset(void* p) { ((CpuRelocSystem*)p)->core.reset(); }
int cpu_reloc_system_set_relocalisation(void* p, int max_lost_frames) {
    if (max_lost_frames < 0) return -1;
    ((CpuRelocSystem*)p)->core.setRelocalisation(max_lost_frames);
    return 0;
}
// the table of alva_system_set_preset (include/alva_b200.h): 0 DEFAULT, 1 FAST, 2 AVERAGE, 3 ACCURATE; -1 = unknown
int cpu_reloc_system_set_preset(void* p, int preset) {
    static const int cell[4] = {40, 50, 45, 35}, p3p[4] = {1, 1, 0, 0}, clahe[4] = {0, 0, 0, 1};
    static const float ratio[4] = {0.95f, 0.9f, 0.9f, 0.95f};
    if (preset < 0 || preset > 3) return -1;
    CpuRelocSystem* s = (CpuRelocSystem*)p;
    s->be.cell = cell[preset];
    s->core.setPreset(cell[preset], ratio[preset], p3p[preset] != 0);
    const int tx = s->be.w / 50, ty = s->be.h / 50;
    s->be.clahe = clahe[preset] != 0; s->be.clip = 3.f; s->be.tx = tx; s->be.ty = ty;
    return 0;
}
void cpu_reloc_system_set_distortion(void* p, double k1, double k2, double p1, double p2) {
    const double d[4] = {k1, k2, p1, p2};
    ((CpuRelocSystem*)p)->core.setDistortion(d);
}
int cpu_reloc_system_process(void* p, const uint8_t* rgba, double t_ms, double* Twc7) {
    CpuRelocSystem* s = (CpuRelocSystem*)p;
    const int st = s->core.process(rgba, t_ms);
    s->core.cur.Twc.to7(Twc7);
    return st;
}
int cpu_reloc_system_keypoints(void* p, int32_t* ids, float* px, uint8_t* is3d, double* wpt, int cap) {
    CpuRelocSystem* s = (CpuRelocSystem*)p;
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
int cpu_reloc_system_info(void* p, int32_t* out8) {
    CpuRelocSystem* s = (CpuRelocSystem*)p;
    out8[0] = s->core.cur.id; out8[1] = s->core.cur.kfid; out8[2] = s->core.cur.n; out8[3] = s->core.cur.n3d;
    out8[4] = s->core.ready_for_init; out8[5] = s->core.n_kf; out8[6] = s->core.cur.nocc; out8[7] = s->core.n_mp_ids;
    return 0;
}
// {times lost, frames relocalised, matches of the last attempt, PnP inliers of the last attempt, lost now, lost frames,
//  map points in the relocalisation table, its descriptor rows}
int cpu_reloc_system_counters(void* p, int32_t* out8) {
    CpuRelocSystem* s = (CpuRelocSystem*)p;
    out8[0] = s->core.n_lost; out8[1] = s->core.n_relocalised; out8[2] = s->core.reloc_last_matches; out8[3] = s->core.reloc_last_inliers;
    out8[4] = s->core.lost ? 1 : 0; out8[5] = s->core.lost_frames; out8[6] = (int32_t)s->core.reloc_table.mp_id.size();
    out8[7] = (int32_t)(s->core.reloc_table.desc.size() / 32);
    return 0;
}
}
