// Host build of the AugmentPipe coordinate / weight function and of the adjoint's enumeration box
// (long-video-gan_b200/csrc/augment_pipe.cuh). For each case, brute force over every v point and every tap of its
// 7 x 7 window: each xpad point with a non-zero weight must lie in the box the adjoint kernel walks for that point, and
// copy_at must list exactly the xpad indices that reflect onto each x index.
//   nvcc -O2 -std=c++17 -o /tmp/augment_pipe_emul tools/augment_pipe_emul.cu && /tmp/augment_pipe_emul
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include "../long-video-gan_b200/csrc/augment_pipe.cuh"

using namespace lvg::ap;

struct M3 {
    double m[3][3];
};

static M3 mul(const M3& a, const M3& b) {
    M3 r{};
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
            for (int k = 0; k < 3; k++) r.m[i][j] += a.m[i][k] * b.m[k][j];
    return r;
}
static M3 affine(double a, double b, double c, double d, double tx, double ty) { return M3{{{a, b, tx}, {c, d, ty}, {0, 0, 1}}}; }
static M3 scale(double sx, double sy) { return affine(sx, 0, 0, sy, 0, 0); }
static M3 shift(double tx, double ty) { return affine(1, 0, 0, 1, tx, ty); }
static M3 rot(double a) { return affine(cos(a), -sin(a), sin(a), cos(a), 0, 0); }

// the Hz_geom taps: a smooth 12-tap low-pass normalised to sum 1 (the box test does not depend on the values, only on
// which taps are non-zero)
static void filter(float* f) {
    double s = 0;
    for (int k = 0; k < kTaps; k++) s += (f[k] = (float)(sin(M_PI * (k + 0.5) / kTaps) + 0.05 * (k % 3)));
    for (int k = 0; k < kTaps; k++) f[k] = (float)(f[k] / s);
}

struct Case {
    const char* name;
    int h, w;
    M3 g;            // G_inv: output pixel -> input pixel
    bool clamp;      // margins at their clamp (size - 1)
};

static int run(const Case& c, const float* f) {
    // margins as the reference computes them: corners of the frame through G_inv, plus 6 - center, within [0, size - 1]
    const double cx = (c.w - 1) / 2.0, cy = (c.h - 1) / 2.0;
    double mg[4] = {-1e300, -1e300, -1e300, -1e300};
    for (int q = 0; q < 4; q++) {
        const double px = (q == 1 || q == 2) ? cx : -cx, py = q >= 2 ? cy : -cy;
        const double ox = c.g.m[0][0] * px + c.g.m[0][1] * py + c.g.m[0][2], oy = c.g.m[1][0] * px + c.g.m[1][1] * py + c.g.m[1][2];
        mg[0] = fmax(mg[0], -ox), mg[1] = fmax(mg[1], -oy), mg[2] = fmax(mg[2], ox), mg[3] = fmax(mg[3], oy);
    }
    int m[4];
    for (int k = 0; k < 4; k++) {
        const double lim = (k % 2 ? c.h : c.w) - 1;
        m[k] = c.clamp ? (int)lim : (int)ceil(fmin(fmax(mg[k] + 6 - (k % 2 ? cy : cx), 0.0), lim));
    }
    const int mx0 = m[0], my0 = m[1], mx1 = m[2], my1 = m[3];
    const int hp = c.h + my0 + my1, wp = c.w + mx0 + mx1, luy = 2 * hp, lux = 2 * wp, hv = 2 * c.h + 12, wv = 2 * c.w + 12;
    M3 g = mul(shift((mx0 - mx1) / 2.0, (my0 - my1) / 2.0), c.g);
    g = mul(mul(scale(2, 2), g), scale(0.5, 0.5));
    g = mul(mul(shift(-0.5, -0.5), g), shift(0.5, 0.5));
    g = mul(mul(scale(2.0 / lux, 2.0 / luy), g), scale(wv / 2.0, hv / 2.0));
    const float th[6] = {(float)g.m[0][0], (float)g.m[0][1], (float)g.m[0][2], (float)g.m[1][0], (float)g.m[1][1], (float)g.m[1][2]};

    int bad = 0;
    long nonzero = 0, walked = 0;
    for (int vi = 0; vi < hv; vi++) {
        for (int vj = 0; vj < wv; vj++) {
            float ix, iy;
            point_coord(th, grid_base(vj, wv), grid_base(vi, hv), lux, luy, ix, iy);
            const Axis ax = axis_of(ix, lux), ay = axis_of(iy, luy);
            for (int ky = 0; ky < kWin; ky++) {
                const int py = ay.i0 + ky;
                if (py < 0 || py >= hp || tap(ay, ky, f) == 0.f) continue;
                for (int kx = 0; kx < kWin; kx++) {
                    const int px = ax.i0 + kx;
                    if (px < 0 || px >= wp || tap(ax, kx, f) == 0.f) continue;
                    nonzero++;
                    const Box b = box_rows(th, px, py, lux, luy, hv);
                    int jl = 0, jh = -1;
                    const bool row = vi >= b.vi_lo && vi <= b.vi_hi && box_cols(th, b, grid_base(vi, hv), wv, jl, jh);
                    if (!row || vj < jl || vj > jh) {
                        if (bad++ < 5)
                            printf("  %s: v point (%d, %d) with a non-zero weight on xpad (%d, %d) is outside its box rows [%d, %d] cols [%d, %d]\n",
                                   c.name, vi, vj, py, px, b.vi_lo, b.vi_hi, jl, jh);
                    }
                }
            }
        }
    }
    // the boxes' total size over all xpad points (what the adjoint walks) against the non-zero weights
    for (int py = 0; py < hp; py++)
        for (int px = 0; px < wp; px++) {
            const Box b = box_rows(th, px, py, lux, luy, hv);
            for (int vi = b.vi_lo; vi <= b.vi_hi; vi++) {
                int jl, jh;
                if (box_cols(th, b, grid_base(vi, hv), wv, jl, jh)) walked += jh - jl + 1;
            }
        }
    // copy_at lists exactly the xpad indices that reflect onto each x index
    for (int axis = 0; axis < 2; axis++) {
        const int len = axis ? c.h : c.w, m0 = axis ? my0 : mx0, m1 = axis ? my1 : mx1;
        for (int j = 0; j < len; j++) {
            int expect = 0, listed = 0;
            for (int i = 0; i < len + m0 + m1; i++) expect += reflect(i, m0, len) == j;
            for (int a = 0; a < 3; a++) {
                const int i = copy_at(j, m0, m1, len, a);
                if (i < 0) continue;
                listed++;
                if (i >= len + m0 + m1 || reflect(i, m0, len) != j) bad++;
            }
            if (listed != expect) bad++;
        }
    }
    printf("%-22s h=%3d w=%3d margins %3d %3d %3d %3d  non-zero weights %9ld  walked %10ld  %s\n", c.name, c.h, c.w, mx0, my0, mx1, my1,
           nonzero, walked, bad ? "FAIL" : "ok");
    return bad;
}

int main() {
    float f[kTaps];
    filter(f);
    std::vector<Case> cases;
    const M3 id = scale(1, 1);
    cases.push_back({"identity", 9, 15, id, false});
    cases.push_back({"identity_clamped", 9, 15, id, true});
    cases.push_back({"rot45", 13, 21, rot(M_PI / 4), false});
    cases.push_back({"rot45_clamped", 13, 21, rot(M_PI / 4), true});
    cases.push_back({"scale_0.25", 9, 15, scale(0.25, 0.25), false});
    cases.push_back({"scale_4", 9, 15, scale(4, 4), false});
    cases.push_back({"scale_4_rot30", 11, 17, mul(rot(0.52), scale(4, 4)), true});
    cases.push_back({"aniso", 12, 20, mul(rot(-1.1), mul(scale(2.3, 1 / 2.3), rot(0.7))), false});
    cases.push_back({"aniso_0.25_4", 12, 20, scale(0.25, 4), false});
    for (int flip = 0; flip < 2; flip++)
        for (int r90 = 0; r90 < 4; r90++) {
            static char names[8][32];
            snprintf(names[flip * 4 + r90], 32, "xflip%d_rot90x%d", flip, r90);
            // rotate2d(pi/2 i) in fp32 leaves cos = -4.4e-8 rather than 0: keep that
            const float cs = cosf((float)(M_PI / 2) * r90), sn = sinf((float)(M_PI / 2) * r90);
            cases.push_back({names[flip * 4 + r90], 9, 15, mul(scale(flip ? -1 : 1, 1), affine(cs, -sn, sn, cs, 0, 0)), r90 == 3});
        }
    srand(7);
    for (int k = 0; k < 12; k++) {
        static char names[12][32];
        snprintf(names[k], 32, "random_%d", k);
        auto u = [] { return (double)rand() / RAND_MAX; };
        const double s = exp2((u() * 2 - 1) * 2), a = exp2((u() * 2 - 1) * 1), t0 = (u() * 2 - 1) * M_PI, t1 = (u() * 2 - 1) * M_PI;
        const int h = 7 + rand() % 30, w = 7 + rand() % 40;
        const M3 g = mul(mul(mul(mul(rot(t0), scale(s, s)), scale(a, 1 / a)), rot(t1)), shift((u() - 0.5) * w * 0.25, (u() - 0.5) * h * 0.25));
        cases.push_back({names[k], h, w, g, k % 3 == 0});
    }
    cases.push_back({"train_shape_rot", 144, 256, mul(rot(0.3), scale(1.1, 0.9)), false});
    int bad = 0;
    for (const Case& c : cases) bad += run(c, f) != 0;
    printf(bad ? "%d cases FAILED\n" : "all ok\n", bad);
    return bad ? 1 : 0;
}
