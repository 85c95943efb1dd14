// fast_swar.h -- the FAST-9 candidate pre-test of the fused front end with ANTIPODAL FLAG SHARING (experimental, opt-in:
// alva_set_option("frontend_antipodal", 1); the default path is fast_candidates8 in frontend.cu).
//
// The pre-test needs, per pixel p and ring offset o, the flag |I(p + o) - I(p)| > t.  The same absolute difference serves pixel
// p at offset o and pixel p + o at offset -o, so only the 8 offsets with dy >= 0 are computed (VABSDIFF4 + carry compare +
// IMAD.HI packing, as before); the 8 antipodal flag words are assembled from them: a byte permute across the neighbouring lane's
// packed word for the column shift (one SHFL + one PRMT) and a per-byte bit shift for the row shift.  A warp holds 8 rows, so
// the first dy rows of an antipodal element have their source outside the warp's rows and are still computed directly (15 of 64
// element-rows).  Per thread: 8 x 8 + 15 = 79 element-rows instead of 128, + 8 x ~4 assembly instructions.
//
// Layout (as frontend.cu): a lane owns one 32-bit word = 4 horizontally adjacent pixels, over 8 consecutive rows; result / flag
// words carry bit 8 j + i for pixel j (byte), row i.  Ring numbering (OpenCV's): 0 (0,+3) 1 (+1,+3) 2 (+2,+2) 3 (+3,+1) 4 (+3,0)
// 5 (+3,-1) 6 (+2,-2) 7 (+1,-3) 8 (0,-3) 9 (-1,-3) 10 (-2,-2) 11 (-3,-1) 12 (-3,0) 13 (-3,+1) 14 (-2,+2) 15 (-1,+3), dy > 0 = rows below.
// Direct set {0, 1, 2, 3, 4, 13, 14, 15}; element m = o ^ 8 is assembled from direct o: flag(p, -o) = D_o(p - o).
//
// Single source for the device and for the HOST EMULATION the CPU suite runs (tests/host/fast_swar_host.cpp emulates the warp with
// arrays and checks this variant against the baseline formulation and against the scalar definition of the pre-test).
#pragma once
#include <stdint.h>

#if defined(__CUDA_ARCH__)
#define FSW_FN __device__ __forceinline__
#define FSW_MEM __device__ __forceinline__
#define FSW_VABSDIFF4(a, b) __vabsdiffu4((a), (b))
#define FSW_PRMT(a, b, s) __byte_perm((a), (b), (s))
FSW_FN uint32_t fsw_madhi(uint32_t u, uint32_t mul, uint32_t acc) { asm("mad.hi.u32 %0, %1, %2, %0;" : "+r"(acc) : "r"(u), "r"(mul)); return acc; }
#else
#define FSW_FN static inline
#define FSW_MEM inline
FSW_FN uint32_t FSW_VABSDIFF4(uint32_t a, uint32_t b) {
    uint32_t r = 0;
    for (int j = 0; j < 4; j++) { const int x = (a >> (8 * j)) & 255, y = (b >> (8 * j)) & 255; r |= (uint32_t)(x > y ? x - y : y - x) << (8 * j); }
    return r;
}
FSW_FN uint32_t FSW_PRMT(uint32_t a, uint32_t b, uint32_t s) {
    const uint64_t v = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int j = 0; j < 4; j++) r |= (uint32_t)((v >> (8 * ((s >> (4 * j)) & 7))) & 255) << (8 * j);
    return r;
}
FSW_FN uint32_t fsw_madhi(uint32_t u, uint32_t mul, uint32_t acc) { return acc + (uint32_t)(((uint64_t)u * mul) >> 32); }
#endif

namespace fast_swar {

// ring offsets as constexpr FUNCTIONS (namespace-scope constexpr arrays are not visible to device code):
// dx = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1}, dy(k) = dx(k + 4)
constexpr int dx_of(int k) { return (k & 15) < 4 ? (k & 15) : (k & 15) < 6 ? 3 : (k & 15) < 12 ? 8 - (k & 15) : (k & 15) < 14 ? -3 : (k & 15) - 16; }
constexpr int dy_of(int k) { return dx_of(k + 4); }
constexpr bool is_direct(int k) { return dy_of(k) > 0 || (dy_of(k) == 0 && dx_of(k) > 0); }   // {0,1,2,3,4,13,14,15}
constexpr int source_of(int m) { return m ^ 8; }                                        // the antipodal (direct) element
constexpr int missing_rows(int m) { return dy_of(source_of(m)); }                          // rows i < dy have no source row in the warp

template <bool HI_THR>
FSW_FN uint32_t absdiff_gt(uint32_t ring, uint32_t c, uint32_t K) {   // bit 7 of byte j = |ring_j - c_j| > t
    const uint32_t a = FSW_VABSDIFF4(ring, c);
    const uint32_t sum = (a & 0x7f7f7f7fu) + K;
    return HI_THR ? (sum & a & 0x80808080u) : ((sum | a) & 0x80808080u);
}

// ring word of element k for the centre row `cr` of a 7-row window (L / M / R = the words left of, at, right of the lane's word)
template <int K>
FSW_FN uint32_t ring_word(const uint32_t* Lw, const uint32_t* Mw, const uint32_t* Rw, int cr) {
    const int r = (cr + dy_of(K) + 7) % 7;   // the caller keeps window row (y mod 7)
    if (dx_of(K) == 0) return Mw[r];
    if (dx_of(K) == 1) return FSW_PRMT(Mw[r], Rw[r], 0x4321);
    if (dx_of(K) == 2) return FSW_PRMT(Mw[r], Rw[r], 0x5432);
    if (dx_of(K) == 3) return FSW_PRMT(Mw[r], Rw[r], 0x6543);
    if (dx_of(K) == -1) return FSW_PRMT(Lw[r], Mw[r], 0x6543);
    if (dx_of(K) == -2) return FSW_PRMT(Lw[r], Mw[r], 0x5432);
    return FSW_PRMT(Lw[r], Mw[r], 0x4321);
}

// phase 1 (per lane): the packed flag words of the direct elements over the 8 rows, and the first `missing_rows` rows of the others.
// g0: the lane's word in the first of the 14 gray rows involved (rows 0..13: centre rows 3..10); pitch in words.
template <bool HI_THR, int PITCH_W, int K, int I>
struct Phase1Elem {
    static FSW_MEM void run(const uint32_t* Lw, const uint32_t* Mw, const uint32_t* Rw, uint32_t c, uint32_t Kc, const uint32_t* mul, uint32_t* acc) {
        if (is_direct(K) || I < missing_rows(K)) {
            const uint32_t U = absdiff_gt<HI_THR>(ring_word<K>(Lw, Mw, Rw, (I + 3) % 7), c, Kc);
            acc[K] = I < 7 ? fsw_madhi(U, mul[I], acc[K]) : acc[K] + U;   // bit 7 of byte j -> bit 8 j + I
        }
        Phase1Elem<HI_THR, PITCH_W, K + 1, I>::run(Lw, Mw, Rw, c, Kc, mul, acc);
    }
};
template <bool HI_THR, int PITCH_W, int I>
struct Phase1Elem<HI_THR, PITCH_W, 16, I> {
    static FSW_MEM void run(const uint32_t*, const uint32_t*, const uint32_t*, uint32_t, uint32_t, const uint32_t*, uint32_t*) {}
};
template <bool HI_THR, int PITCH_W, int I>
struct Phase1Row {
    static FSW_MEM void run(const uint32_t* g0, uint32_t* Lw, uint32_t* Mw, uint32_t* Rw, uint32_t Kc, const uint32_t* mul, uint32_t* acc) {
        constexpr int r = I + 6;   // bring in window row i + 6; rows i .. i + 6 <-> dy = -3 .. +3 around centre row i + 3
        Lw[r % 7] = g0[r * PITCH_W - 1]; Mw[r % 7] = g0[r * PITCH_W]; Rw[r % 7] = g0[r * PITCH_W + 1];
        Phase1Elem<HI_THR, PITCH_W, 0, I>::run(Lw, Mw, Rw, Mw[(I + 3) % 7], Kc, mul, acc);
        Phase1Row<HI_THR, PITCH_W, I + 1>::run(g0, Lw, Mw, Rw, Kc, mul, acc);
    }
};
template <bool HI_THR, int PITCH_W>
struct Phase1Row<HI_THR, PITCH_W, 8> {
    static FSW_MEM void run(const uint32_t*, uint32_t*, uint32_t*, uint32_t*, uint32_t, const uint32_t*, uint32_t*) {}
};

template <bool HI_THR, int PITCH_W>
FSW_FN void phase1(const uint32_t* g0, uint32_t Kc, const uint32_t* mul, uint32_t* acc) {
    uint32_t Lw[7], Mw[7], Rw[7];
    for (int k = 0; k < 16; k++) acc[k] = 0u;
    for (int r = 0; r < 6; r++) { Lw[r] = g0[r * PITCH_W - 1]; Mw[r] = g0[r * PITCH_W]; Rw[r] = g0[r * PITCH_W + 1]; }
    Phase1Row<HI_THR, PITCH_W, 0>::run(g0, Lw, Mw, Rw, Kc, mul, acc);
}

// phase 2 (per lane): element m from its antipodal direct element o = m ^ 8: flag(p, m) = D_o(p - o).  own / left / right = the
// packed word of element o in this lane and in the lanes holding the 4 pixels to the left / right.
template <int M>
FSW_FN uint32_t assemble(uint32_t own, uint32_t left, uint32_t right, uint32_t partial) {
    constexpr int o = source_of(M), dx = dx_of(o), dy = dy_of(o);
    uint32_t W;
    if (dx == 0) W = own;
    else if (dx == 1) W = FSW_PRMT(left, own, 0x6543);    // byte j <- pixel j - 1
    else if (dx == 2) W = FSW_PRMT(left, own, 0x5432);
    else if (dx == 3) W = FSW_PRMT(left, own, 0x4321);
    else if (dx == -1) W = FSW_PRMT(own, right, 0x4321);  // byte j <- pixel j + 1
    else if (dx == -2) W = FSW_PRMT(own, right, 0x5432);
    else W = FSW_PRMT(own, right, 0x6543);
    constexpr uint32_t keep = ((0xffu << dy) & 0xffu) * 0x01010101u;   // rows >= dy of every byte; row i <- source row i - dy
    return ((W << dy) & keep) | partial;
}

// the 9-of-16 contiguity network on the 16 packed flag words (as in frontend.cu)
FSW_FN uint32_t contiguous9(const uint32_t* acc) {
    uint32_t T[16];
    for (int k = 0; k < 16; k++) T[k] = acc[k] & acc[(k + 1) & 15] & acc[(k + 2) & 15];
    uint32_t cand = 0;
    for (int k = 0; k < 16; k++) cand |= T[k] & T[(k + 3) & 15] & T[(k + 6) & 15];
    return cand;
}

}  // namespace fast_swar
