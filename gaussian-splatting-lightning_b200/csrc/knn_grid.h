// Sizing of the k-NN hash grid from the points' bounding box (knn.cu runs it in one device thread).  Plain C++ as well as CUDA, so
// tests/test_similarity_reg_cpu.py compiles it with the host compiler and checks it on boxes no GPU should ever be handed.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define B200GS_HD __host__ __device__
#else
#define B200GS_HD
#endif

namespace b200gs {

struct KnnGrid {
    float lox, loy, loz, cs, inv_cs;
    int gx, gy, gz;
};

constexpr int GRID_AXIS_MAX = 1024;
constexpr int GRID_SIZING_STEPS = 64;   // from a start within the per-axis cap, 1.26^26 > 1023 / 3 reaches 4^3 <= 64 <= max_cells cells

// lo / hi: the bounding box of the points with finite coordinates; an axis with lo > hi, or a non-finite bound (no finite points),
// gets one cell at 0.  About two points per OCCUPIED-volume cell (flat or linear point sets fall back to their largest extent), at
// most GRID_AXIS_MAX cells per axis and max_cells (>= 64) in total.  Extents are formed in double, so boxes whose float width
// overflows (-3e38 .. 3e38) stay finite, and the cell size starts where every axis is within the cap: the loop that grows it runs at
// most GRID_SIZING_STEPS times, and a grid that still has too many cells falls back to a single cell.
B200GS_HD inline KnnGrid size_knn_grid(const float lo[3], const float hi[3], int64_t n, int64_t max_cells) {
    double base[3], ext[3], emax = 0.0;
    for (int a = 0; a < 3; ++a) {
        const bool ok = isfinite(lo[a]) && isfinite(hi[a]) && lo[a] <= hi[a];
        base[a] = ok ? (double)lo[a] : 0.0;
        ext[a] = ok ? (double)hi[a] - (double)lo[a] : 0.0;
        emax = fmax(emax, ext[a]);
    }
    const double vol = fmax(ext[0], 1e-3 * emax) * fmax(ext[1], 1e-3 * emax) * fmax(ext[2], 1e-3 * emax);
    double cs = emax > 0.0 ? fmax(cbrt(vol / (0.5 * (double)(n > 0 ? n : 1))), emax / (GRID_AXIS_MAX - 1)) : 1.0;
    if (!(cs > 0.0) || !isfinite(cs)) cs = 1.0;
    int g[3] = {1, 1, 1};
    bool fits = false;
    for (int step = 0; step < GRID_SIZING_STEPS && !fits; ++step) {
        for (int a = 0; a < 3; ++a) g[a] = (int)fmin((double)GRID_AXIS_MAX, floor(ext[a] / cs) + 1.0);
        fits = (int64_t)g[0] * g[1] * g[2] <= max_cells;
        if (!fits) cs *= 1.26;
    }
    if (!fits) {
        g[0] = g[1] = g[2] = 1;
        cs = fmax(emax, 1.0);
    }
    KnnGrid out;
    out.lox = (float)base[0];
    out.loy = (float)base[1];
    out.loz = (float)base[2];
    out.cs = (float)fmin(fmax(cs, 1e-30), 3.0e38);   // a normal float whose reciprocal is finite
    out.inv_cs = (float)(1.0 / (double)out.cs);
    out.gx = g[0];
    out.gy = g[1];
    out.gz = g[2];
    return out;
}

}  // namespace b200gs
