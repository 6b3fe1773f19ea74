// Projection and GridStructure cell helpers shared by the batched pipeline's frame-to-frame geometry (pipeline.cu,
// k_mg_geom_f2f) and the keyframe / local-map matchers (kfmatch.cu).
#pragma once

#define PLF_GRID_ROWS 48   // stvo-pl gridStructure.h (SURVEY Appendix A.2)
#define PLF_GRID_COLS 64

__device__ __forceinline__ int mg_cell(double v) { return (int)v; }   // double -> int as in C++ (truncation)

// The cell of a projected query coordinate.  The reference converts with a plain double -> int, undefined for NaN and
// beyond int range; the library defines both: NaN (a point at infinity projects to inf / inf) -> 0, and values clamped
// to +-2^28, which keeps Bresenham differences inside int (oracle/frontend.py _cell).
#define PLF_CELL_LIM 268435456.0
__device__ __forceinline__ int plf_qcell(double v) {
  if (v != v) return 0;
  return mg_cell(fmin(fmax(v, -PLF_CELL_LIM), PLF_CELL_LIM));
}

// PinholeStereoCamera::projection: (cx + fx X / Z, cy + fy Y / Z), per coordinate and for both
__device__ __forceinline__ double plf_project_u(double fx, double cx, double X, double Z) { return cx + fx * X / Z; }
__device__ __forceinline__ double plf_project_v(double fy, double cy, double Y, double Z) { return cy + fy * Y / Z; }
__device__ __forceinline__ double2 plf_project(double fx, double fy, double cx, double cy, double X, double Y, double Z) {
  return make_double2(plf_project_u(fx, cx, X, Z), plf_project_v(fy, cy, Y, Z));
}

// A train line of the windowed matcher (src/mapHandler.cpp:400-411, :688-699): the cells of its scaled end points and
// its normalised scaled direction (unguarded like the reference's normalize()).
__device__ __forceinline__ void plf_train_line(double2 sp, double2 ep, double iw, double ih, int* d, double* dir) {
  d[0] = mg_cell(sp.x * iw); d[1] = mg_cell(sp.y * ih); d[2] = mg_cell(ep.x * iw); d[3] = mg_cell(ep.y * ih);
  const double vx = (ep.x - sp.x) * iw, vy = (ep.y - sp.y) * ih, nrm = sqrt(vx * vx + vy * vy);
  dir[0] = vx / nrm;
  dir[1] = vy / nrm;
}
