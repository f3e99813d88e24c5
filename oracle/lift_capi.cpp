// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header).  C entry points of the restated hash-to-curve and initial global cumulative
// sum (lift.hpp), built into their own library, oracle/libliftoracle.so (oracle/lift.mk), for tests/lift_oracle_lib.py.  Field elements
// cross as u32 Montgomery words.
#include "lift.hpp"
#include <cstring>

using namespace orc;

static S7 ld7(const uint32_t* p) { S7 r; for (int i = 0; i < 7; i++) r.c[i] = F::raw(p[i]); return r; }
static void st7(const S7& a, uint32_t* p) { for (int i = 0; i < 7; i++) p[i] = a.c[i].v; }

extern "C" {
// lift_x of n messages (8 Montgomery words each) -> offsets[i] (-1 where the reference panics) and the points (14 words)
void orc_lift_x(const uint32_t* msgs, int32_t* offsets, uint32_t* pts, uint64_t n) {
#pragma omp parallel for schedule(dynamic, 16)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        F m[8];
        for (int k = 0; k < 8; k++) m[k] = F::raw(msgs[8 * i + k]);
        SPoint p;
        offsets[i] = lift_x(m, p);
        if (offsets[i] >= 0) { st7(p.x, pts + 14 * i); st7(p.y, pts + 14 * i + 7); }
    }
}
// SepticExtension::sqrt of n elements -> ok[i] = 0 for a non-square
void orc_septic_sqrt(const uint32_t* a, uint32_t* out, uint32_t* ok, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        S7 r;
        ok[i] = s7_sqrt(ld7(a + 7 * i), r);
        if (ok[i]) st7(r, out + 7 * i);
    }
}
// SepticCurveComplete + of n point pairs; infinity = 14 zero words
void orc_curve_add_complete(const uint32_t* p, const uint32_t* q, uint32_t* out, uint64_t n) {
    auto ld = [](const uint32_t* w) {
        CPoint c;
        for (int k = 0; k < 14; k++) c.inf = c.inf && w[k] == 0;
        c.p = SPoint{ld7(w), ld7(w + 7)};
        return c;
    };
    for (uint64_t i = 0; i < n; i++) {
        const CPoint r = c_add(ld(p + 14 * i), ld(q + 14 * i));
        if (r.inf) memset(out + 14 * i, 0, 56);
        else { st7(r.p.x, out + 14 * i); st7(r.p.y, out + 14 * i + 7); }
    }
}
// Program::initial_global_cumulative_sum -> 0 and out14, 1 (an entry without a point: *bad), 2 (the sum is at infinity)
int orc_initial_global_cumulative_sum(const uint64_t* addrs, const uint64_t* words, uint64_t n_mem, const uint64_t* pages, const uint8_t* prots,
                                      uint64_t n_pages, int untrusted, uint32_t* out14, uint64_t* bad) {
    SPoint s;
    const int r = initial_global_cumulative_sum(addrs, words, n_mem, pages, prots, n_pages, untrusted != 0, s, bad);
    if (r == 0) { st7(s.x, out14); st7(s.y, out14 + 7); }
    return r;
}
}
