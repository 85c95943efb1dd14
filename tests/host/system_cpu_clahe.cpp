// tests/host/system_cpu_clahe.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libalva_b200.so).
// The CPU oracle build of the System state machine (system_cpu_backend.cpp) with the reference's CLAHE pre-processing switch:
// VisualFrontend::preprocessImage equalises the gray frame before it builds the KLT pyramid (visual_frontend.cpp:672-698), the
// grid detector reads that equalised image (map_manager.cpp:213) and ORB describes the RAW gray frame (map_manager.cpp:204, 218).
// With CLAHE off it is exactly the backend of system_cpu_backend.cpp.  C entry points: cpu_clahe_system_*, one per
// cpu_system_* of that file, plus cpu_system_set_clahe.
#include "system_cpu_backend.cpp"

// orc_clahe: oracle/clahe_oracle.c (linked from tests/_build/libclahe_oracle.so, tests/clahe_util.py)
extern "C" int orc_clahe(const uint8_t* src, uint8_t* dst, int w, int h, int nframes, double clip_limit, int tiles_x, int tiles_y);

struct CpuClaheBackend : CpuBackend {
    bool clahe = false;
    float clip = 3.f;   // State::claheContrastLimit_ is a float (state.hpp:44)
    int tx = 0, ty = 0;
    std::vector<uint8_t> raw;

    int pyramid(const uint8_t* rgba) {
        if (!clahe) return CpuBackend::pyramid(rgba);
        cur ^= 1;
        raw.resize((size_t)w * h);
        orc_gray(rgba, w, h, raw.data());
        orc_clahe(raw.data(), img[cur][0].data(), w, h, 1, (double)clip, tx, ty);
        for (int k = 1; k < nlev; k++) orc_pyrdown(img[cur][k - 1].data(), lw[k - 1], lh[k - 1], img[cur][k].data());
        for (int k = 0; k < nlev; k++) orc_scharr(img[cur][k].data(), lw[k], lh[k], der[cur][k].data());
        blur_valid = false;
        return 0;
    }
    int describe(const float* pts, int n, uint8_t* desc, uint8_t* kept) {
        if (!clahe) return CpuBackend::describe(pts, n, desc, kept);
        if (!blur_valid) { orc_orb_blur(raw.data(), w, h, 0, blur.data()); blur_valid = true; }
        orc_orb_describe(blur.data(), w, h, pts, nullptr, n, desc, kept);
        return 0;
    }
};

struct CpuClaheSystem {
    CpuClaheBackend be;
    alva_sys::SystemCore<CpuClaheBackend> core;
    CpuClaheSystem() : core(be) {}
};

extern "C" {
void* cpu_clahe_system_create(int w, int h, double fx, double fy, double cx, double cy) {
    CpuClaheSystem* s = new CpuClaheSystem();
    s->be.init(w, h);
    s->be.fx = fx; s->be.fy = fy; s->be.cx = cx; s->be.cy = cy;
    s->core.configure(w, h, fx, fy, cx, cy);
    return s;
}
// State::claheEnabled_ / claheContrastLimit_ / claheTileSize_ with VisualFrontend's grid (visual_frontend.cpp:16-18); -1 = empty grid
int cpu_system_set_clahe(void* p, int enabled, double clip_limit, int tile_size) {
    CpuClaheSystem* s = (CpuClaheSystem*)p;
    const int tx = tile_size > 0 ? s->be.w / tile_size : 0, ty = tile_size > 0 ? s->be.h / tile_size : 0;
    if (tx < 1 || ty < 1) return -1;
    s->be.clahe = enabled != 0; s->be.clip = (float)clip_limit; s->be.tx = tx; s->be.ty = ty;
    return 0;
}
void cpu_clahe_system_set_essential_hook(void* p, void* fn) {
    ((CpuClaheSystem*)p)->be.essential_hook = (int (*)(const double*, const double*, int, int, float, int, float, float, double*, uint8_t*))fn;
}
void cpu_clahe_system_destroy(void* p) { delete (CpuClaheSystem*)p; }
int cpu_clahe_system_process(void* p, const uint8_t* rgba, double t_ms, double* Twc7) {
    CpuClaheSystem* s = (CpuClaheSystem*)p;
    const int st = s->core.process(rgba, t_ms);
    s->core.cur.Twc.to7(Twc7);
    return st;
}
int cpu_clahe_system_keypoints(void* p, int32_t* ids, float* px, uint8_t* is3d, double* wpt, int cap) {
    CpuClaheSystem* s = (CpuClaheSystem*)p;
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
int cpu_clahe_system_info(void* p, int32_t* out8) {
    CpuClaheSystem* s = (CpuClaheSystem*)p;
    out8[0] = s->core.cur.id; out8[1] = s->core.cur.kfid; out8[2] = s->core.cur.n; out8[3] = s->core.cur.n3d;
    out8[4] = s->core.ready_for_init; out8[5] = s->core.n_kf; out8[6] = s->core.cur.nocc; out8[7] = s->core.n_mp_ids;
    return 0;
}
}
