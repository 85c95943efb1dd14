/* oracle/clahe_oracle.c -- CPU restatement of the reference's CLAHE pre-processing.
 *
 * TEST INFRASTRUCTURE ONLY (see alva_oracle.c's header): the parity oracle of alva_k_clahe.  Built on demand by the tests
 * (tests/clahe_util.py: gcc -O2 -ffp-contract=off -fPIC -shared into tests/_build/libclahe_oracle.so); pinned bit for bit to the
 * reference's own OpenCV by tests/test_oracle_clahe.py (live through oracle/_ref/libalva_ref_clahe.so, else the digests of
 * tests/golden/clahe.npz).  -ffp-contract=off matters: the interpolation below is fusion-sensitive.
 *
 * CLAHE, 8-bit: cv::createCLAHE(clip_limit, Size(tiles_x, tiles_y))->apply(src, dst) as VisualFrontend::preprocessImage calls
 * it (src/slam/src/visual_frontend.cpp:16-18, 678-681) -> src/libs/opencv/modules/imgproc/src/clahe.cpp, CLAHE_Impl::apply
 * (349-429), CLAHE_CalcLut_Body (142-221), CLAHE_Interpolation_Body (223-313).  nframes tightly packed frames; dst may equal src.
 *  - tiles (clahe.cpp:362-385): w/tx x h/ty when both axes divide; otherwise the LUT source is the image extended at the
 *    bottom / right by tiles - size % tiles on BOTH axes (BORDER_REFLECT_101, an evenly dividing axis by a full `tiles`),
 *    tile = extended size / tiles.  Read here by index.
 *  - clip (clahe.cpp:387-394): (int)(clip_limit * area / 256) in double, at least 1; 0 = none.  An out-of-range conversion
 *    gives INT_MIN on x86 (cvttsd2si), so the max() makes it 1.
 *  - redistribution (clahe.cpp:187-208), LUT (clahe.cpp:211-219): saturate_cast<uchar>(sum * lutScale), lutScale = 255.0f / area
 *    (float), cvRound = round half to even.
 *  - interpolation (clahe.cpp:236-312): float, unfused, in the reference's evaluation order.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

/* cv::borderInterpolate(BORDER_REFLECT_101), repeated reflection included (core/src/copy.cpp) */
static inline int reflect101(int p, int n)
{
    if (n == 1) return 0;
    while (p < 0 || p >= n) {
        if (p < 0) p = -p;
        else p = 2 * (n - 1) - p;
    }
    return p;
}

/* cvRound(float): round-half-to-even (SSE cvtss2si) -- core/include/opencv2/core/fast_math.hpp */
static inline int cv_roundf(float v) { return (int)lrintf(v); }

int orc_clahe_clip(double clip_limit, int area)
{
    if (!(clip_limit > 0.0)) return 0;
    const double v = clip_limit * area / 256;
    const int c = (v >= 2147483648.0 || v <= -2147483649.0) ? INT32_MIN : (int)v;
    return c > 1 ? c : 1;
}

void orc_clahe_lut(const uint8_t* src, int w, int h, int tx, int tw, int th, int clip, int k, uint8_t* lut)
{
    int hist[256];
    memset(hist, 0, sizeof hist);
    const int x0 = (k % tx) * tw, y0 = (k / tx) * th;
    for (int y = y0; y < y0 + th; y++) {
        const uint8_t* row = src + (size_t)reflect101(y, h) * w;
        for (int x = x0; x < x0 + tw; x++) hist[row[reflect101(x, w)]]++;
    }
    if (clip > 0) {
        int clipped = 0;
        for (int i = 0; i < 256; i++)
            if (hist[i] > clip) { clipped += hist[i] - clip; hist[i] = clip; }
        const int batch = clipped / 256;
        int residual = clipped - batch * 256;
        for (int i = 0; i < 256; i++) hist[i] += batch;
        if (residual != 0) {
            const int step = 256 / residual > 1 ? 256 / residual : 1;
            for (int i = 0; i < 256 && residual > 0; i += step, residual--) hist[i]++;
        }
    }
    const float scale = 255.0f / (float)(tw * th);
    int sum = 0;
    for (int i = 0; i < 256; i++) {
        sum += hist[i];
        const int v = cv_roundf((float)sum * scale);
        lut[i] = (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
    }
}

int orc_clahe(const uint8_t* src, uint8_t* dst, int w, int h, int nframes, double clip_limit, int tx, int ty)
{
    if (w < 1 || h < 1 || nframes < 1 || tx < 1 || ty < 1 || tx > w || ty > h || !(clip_limit >= 0.0)) return -1;
    const int even = (w % tx == 0 && h % ty == 0);
    const int tw = even ? w / tx : (w + tx - w % tx) / tx;
    const int th = even ? h / ty : (h + ty - h % ty) / ty;
    const int clip = orc_clahe_clip(clip_limit, tw * th);
    uint8_t* lut = (uint8_t*)malloc((size_t)tx * ty * 256);
    uint8_t* out = (uint8_t*)malloc((size_t)w * h);
    const float inv_tw = 1.0f / (float)tw, inv_th = 1.0f / (float)th;
    for (int f = 0; f < nframes; f++) {
        const uint8_t* s = src + (size_t)f * w * h;
        for (int k = 0; k < tx * ty; k++) orc_clahe_lut(s, w, h, tx, tw, th, clip, k, lut + (size_t)k * 256);
        for (int y = 0; y < h; y++) {
            const float tyf = (float)y * inv_th - 0.5f;
            int ty1 = (int)floorf(tyf), ty2 = ty1 + 1;
            const float ya = tyf - (float)ty1, ya1 = 1.0f - ya;
            ty1 = ty1 > 0 ? ty1 : 0;
            ty2 = ty2 < ty - 1 ? ty2 : ty - 1;
            const uint8_t* L1 = lut + (size_t)ty1 * tx * 256;
            const uint8_t* L2 = lut + (size_t)ty2 * tx * 256;
            for (int x = 0; x < w; x++) {
                const float txf = (float)x * inv_tw - 0.5f;
                int tx1 = (int)floorf(txf), tx2 = tx1 + 1;
                const float xa = txf - (float)tx1, xa1 = 1.0f - xa;
                tx1 = tx1 > 0 ? tx1 : 0;
                tx2 = tx2 < tx - 1 ? tx2 : tx - 1;
                const int v = s[(size_t)y * w + x];
                const int i1 = tx1 * 256 + v, i2 = tx2 * 256 + v;
                const float res = ((float)L1[i1] * xa1 + (float)L1[i2] * xa) * ya1 + ((float)L2[i1] * xa1 + (float)L2[i2] * xa) * ya;
                const int r = cv_roundf(res);
                out[(size_t)y * w + x] = (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
            }
        }
        memcpy(dst + (size_t)f * w * h, out, (size_t)w * h);
    }
    free(lut); free(out);
    return 0;
}
