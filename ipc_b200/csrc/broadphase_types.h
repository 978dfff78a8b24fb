// broadphase_types.h -- POD types shared by host (context.h) and device code (broadphase.cuh)
#pragma once
namespace ipcgpu {
struct Grid {
    double ox, oy, oz, inv_h;
    int nx, ny, nz;
    double q_inv; // 1 / quantisation step of the 16-bit entry boxes (65533 steps over the largest axis span)
};
// one entry of a sorted grid: the primitive's box quantised CONSERVATIVELY to 16 bits per coordinate (lo rounded down, hi rounded up,
// one more step each way against floating-point rounding) + its id: 16 bytes = one 128-bit load per candidate instead of a 48-byte
// double box + a 4-byte id.  The quantised overlap test is a superset of the exact one; membership is decided afterwards by the exact
// filters (classification / reference voxel ranges), so nothing depends on the quantisation.
struct QEntry {
    unsigned short lo[3], hi[3];
    int id;
};
struct Box {
    double lo[3], hi[3];
};
// swept grid of the CCD on the reference voxel lattice (ccd.cu): K x K x K voxels per cell, n cells per axis; lmax / hmax: the longest voxel
// range of any primitive and the largest voxel index per axis, from which K is chosen on the device
struct SweptCells {
    int K, n[3];
    int lmax, hmax[3];
};
} // namespace ipcgpu
