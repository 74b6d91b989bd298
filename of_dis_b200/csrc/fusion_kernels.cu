// Volumetric TSDF fusion (ofdis_fuse_push / ofdis_fuse_extract / ofdis_fuse_render; the header states the contract,
// preprocess.fuse_integrate, fuse_extract and fuse_render restate it bit for bit).  Float32 without contraction.
//   fuse_integrate_kernel  one thread per voxel for the whole call: T, W (and colour) loaded once, the n frames in
//                          order, one store.  The volume's HBM traffic is then 2 x 8 (11) bytes per voxel per call; the
//                          disparity and colour gathers of neighbouring voxels fall on neighbouring pixels and go
//                          through L2.
//   fuse_count_kernel      crossings per scan block of FUSE_BLOCK voxels (4 consecutive voxels per thread);
//   fuse_scan_kernel       one CTA: the blocks' exclusive offsets (64-bit) and the total;
//   fuse_write_kernel      the block's crossings again, scanned within the CTA, written at their global index while it
//                          is below the capacity: the order of the header, whatever the grid.
//   fuse_render_kernel     one thread per (pose, pixel), fixed-step ray march to the first sign change.
// Marching cubes (ofdis_fuse_mesh; preprocess.fuse_mesh restates it): the count, scan and write kernels above give the
// vertices, the write kernel also each crossing voxel's first vertex index, then
//   fuse_cube_count_kernel triangles per scan block of FUSE_BLOCK cubes (cube = the voxel of its corner 0), scanned by
//                          fuse_scan_kernel into a second offset array;
//   fuse_face_kernel       the block's triangles again, written at their global index while it is below the capacity.
#include <cfloat>

#include <cuda_runtime.h>

#include "ofdis_internal.cuh"

namespace ofdis {

namespace {

constexpr int FUSE_THREADS = 256;
constexpr int FUSE_VPT = FUSE_BLOCK / FUSE_THREADS;  // voxels per thread of the count and write kernels
constexpr int FUSE_SCAN_THREADS = 1024;
constexpr int FUSE_RENDER_ROWS = 8;                 // a render CTA is 32 x 8 pixels of one pose

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }

// The marching-cubes table of ofdis_fuse_mesh, as preprocess.fuse_mc_table generates it from the header's rules: row =
// case, [0] the triangles, [1 + 3t + s] the cube edge of triangle t's vertex s, 255 past the last.
__constant__ unsigned char FUSE_MC[256][16] = {
    {0, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 0, 8, 4, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 0, 5, 9, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 4, 5, 8, 5, 9, 8, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 1, 4, 10, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 8, 1, 8, 10, 1, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 5, 9, 1, 4, 10, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 1, 5, 10, 5, 9, 10, 9, 8, 10, 255, 255, 255, 255, 255, 255},
    {1, 1, 11, 5, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 8, 4, 1, 11, 5, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 1, 9, 1, 11, 9, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 1, 11, 4, 11, 9, 4, 9, 8, 4, 255, 255, 255, 255, 255, 255},
    {2, 4, 10, 5, 10, 11, 5, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 5, 8, 10, 5, 10, 11, 5, 255, 255, 255, 255, 255, 255},
    {3, 0, 4, 9, 4, 10, 9, 10, 11, 9, 255, 255, 255, 255, 255, 255},
    {2, 8, 10, 9, 10, 11, 9, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 2, 6, 8, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 2, 4, 2, 6, 4, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 5, 9, 2, 6, 8, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 2, 6, 9, 6, 4, 9, 4, 5, 9, 255, 255, 255, 255, 255, 255},
    {2, 1, 4, 10, 2, 6, 8, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 2, 1, 2, 6, 1, 6, 10, 1, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 9, 1, 4, 10, 2, 6, 8, 255, 255, 255, 255, 255, 255},
    {4, 1, 5, 10, 5, 9, 10, 9, 2, 10, 2, 6, 10, 255, 255, 255},
    {2, 1, 11, 5, 2, 6, 8, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 2, 4, 2, 6, 4, 1, 11, 5, 255, 255, 255, 255, 255, 255},
    {3, 0, 1, 9, 1, 11, 9, 2, 6, 8, 255, 255, 255, 255, 255, 255},
    {4, 1, 11, 4, 11, 9, 4, 9, 2, 4, 2, 6, 4, 255, 255, 255},
    {3, 2, 6, 8, 4, 10, 5, 10, 11, 5, 255, 255, 255, 255, 255, 255},
    {4, 0, 2, 5, 2, 6, 5, 6, 10, 5, 10, 11, 5, 255, 255, 255},
    {4, 0, 4, 9, 4, 10, 9, 10, 11, 9, 2, 6, 8, 255, 255, 255},
    {3, 2, 6, 9, 6, 10, 9, 10, 11, 9, 255, 255, 255, 255, 255, 255},
    {1, 2, 9, 7, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 8, 4, 2, 9, 7, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 5, 2, 5, 7, 2, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 2, 8, 7, 8, 4, 7, 4, 5, 7, 255, 255, 255, 255, 255, 255},
    {2, 1, 4, 10, 2, 9, 7, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 1, 8, 10, 1, 2, 9, 7, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 2, 5, 7, 2, 1, 4, 10, 255, 255, 255, 255, 255, 255},
    {4, 1, 5, 10, 5, 7, 10, 7, 2, 10, 2, 8, 10, 255, 255, 255},
    {2, 1, 11, 5, 2, 9, 7, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 4, 1, 11, 5, 2, 9, 7, 255, 255, 255, 255, 255, 255},
    {3, 0, 1, 2, 1, 11, 2, 11, 7, 2, 255, 255, 255, 255, 255, 255},
    {4, 1, 11, 4, 11, 7, 4, 7, 2, 4, 2, 8, 4, 255, 255, 255},
    {3, 2, 9, 7, 4, 10, 5, 10, 11, 5, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 5, 8, 10, 5, 10, 11, 5, 2, 9, 7, 255, 255, 255},
    {4, 0, 4, 2, 4, 10, 2, 10, 11, 2, 11, 7, 2, 255, 255, 255},
    {3, 2, 8, 7, 8, 10, 7, 10, 11, 7, 255, 255, 255, 255, 255, 255},
    {2, 6, 8, 7, 8, 9, 7, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 9, 4, 9, 7, 4, 7, 6, 4, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 8, 5, 7, 8, 7, 6, 8, 255, 255, 255, 255, 255, 255},
    {2, 4, 5, 6, 5, 7, 6, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 1, 4, 10, 6, 8, 7, 8, 9, 7, 255, 255, 255, 255, 255, 255},
    {4, 0, 9, 1, 9, 7, 1, 7, 6, 1, 6, 10, 1, 255, 255, 255},
    {4, 0, 5, 8, 5, 7, 8, 7, 6, 8, 1, 4, 10, 255, 255, 255},
    {3, 1, 5, 10, 5, 7, 10, 7, 6, 10, 255, 255, 255, 255, 255, 255},
    {3, 1, 11, 5, 6, 8, 7, 8, 9, 7, 255, 255, 255, 255, 255, 255},
    {4, 0, 9, 4, 9, 7, 4, 7, 6, 4, 1, 11, 5, 255, 255, 255},
    {4, 0, 1, 8, 1, 11, 8, 11, 7, 8, 7, 6, 8, 255, 255, 255},
    {3, 1, 11, 4, 11, 7, 4, 7, 6, 4, 255, 255, 255, 255, 255, 255},
    {4, 4, 10, 5, 10, 11, 5, 6, 8, 7, 8, 9, 7, 255, 255, 255},
    {5, 0, 6, 5, 0, 9, 6, 9, 7, 6, 6, 10, 5, 10, 11, 5},
    {5, 0, 11, 8, 0, 4, 11, 4, 10, 11, 11, 7, 8, 7, 6, 8},
    {2, 6, 10, 7, 10, 11, 7, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 3, 10, 6, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 8, 4, 3, 10, 6, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 5, 9, 3, 10, 6, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 3, 10, 6, 4, 5, 8, 5, 9, 8, 255, 255, 255, 255, 255, 255},
    {2, 1, 4, 3, 4, 6, 3, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 1, 8, 6, 1, 6, 3, 1, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 9, 1, 4, 3, 4, 6, 3, 255, 255, 255, 255, 255, 255},
    {4, 1, 5, 3, 5, 9, 3, 9, 8, 3, 8, 6, 3, 255, 255, 255},
    {2, 1, 11, 5, 3, 10, 6, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 4, 1, 11, 5, 3, 10, 6, 255, 255, 255, 255, 255, 255},
    {3, 0, 1, 9, 1, 11, 9, 3, 10, 6, 255, 255, 255, 255, 255, 255},
    {4, 1, 11, 4, 11, 9, 4, 9, 8, 4, 3, 10, 6, 255, 255, 255},
    {3, 3, 11, 6, 11, 5, 6, 5, 4, 6, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 5, 8, 6, 5, 6, 3, 5, 3, 11, 5, 255, 255, 255},
    {4, 0, 4, 9, 4, 6, 9, 6, 3, 9, 3, 11, 9, 255, 255, 255},
    {3, 3, 11, 6, 11, 9, 6, 9, 8, 6, 255, 255, 255, 255, 255, 255},
    {2, 2, 3, 8, 3, 10, 8, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 2, 4, 2, 3, 4, 3, 10, 4, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 9, 2, 3, 8, 3, 10, 8, 255, 255, 255, 255, 255, 255},
    {4, 2, 3, 9, 3, 10, 9, 10, 4, 9, 4, 5, 9, 255, 255, 255},
    {3, 1, 4, 3, 4, 8, 3, 8, 2, 3, 255, 255, 255, 255, 255, 255},
    {2, 0, 2, 1, 2, 3, 1, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {4, 0, 5, 9, 1, 4, 3, 4, 8, 3, 8, 2, 3, 255, 255, 255},
    {3, 1, 5, 3, 5, 9, 3, 9, 2, 3, 255, 255, 255, 255, 255, 255},
    {3, 1, 11, 5, 2, 3, 8, 3, 10, 8, 255, 255, 255, 255, 255, 255},
    {4, 0, 2, 4, 2, 3, 4, 3, 10, 4, 1, 11, 5, 255, 255, 255},
    {4, 0, 1, 9, 1, 11, 9, 2, 3, 8, 3, 10, 8, 255, 255, 255},
    {5, 1, 11, 4, 11, 9, 4, 9, 2, 4, 2, 3, 4, 3, 10, 4},
    {4, 2, 3, 8, 3, 11, 8, 11, 5, 8, 5, 4, 8, 255, 255, 255},
    {3, 0, 2, 5, 2, 3, 5, 3, 11, 5, 255, 255, 255, 255, 255, 255},
    {5, 0, 4, 9, 4, 3, 9, 4, 8, 3, 8, 2, 3, 3, 11, 9},
    {2, 2, 3, 9, 3, 11, 9, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 2, 9, 7, 3, 10, 6, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 4, 2, 9, 7, 3, 10, 6, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 2, 5, 7, 2, 3, 10, 6, 255, 255, 255, 255, 255, 255},
    {4, 2, 8, 7, 8, 4, 7, 4, 5, 7, 3, 10, 6, 255, 255, 255},
    {3, 1, 4, 3, 4, 6, 3, 2, 9, 7, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 1, 8, 6, 1, 6, 3, 1, 2, 9, 7, 255, 255, 255},
    {4, 0, 5, 2, 5, 7, 2, 1, 4, 3, 4, 6, 3, 255, 255, 255},
    {5, 1, 5, 3, 5, 8, 3, 5, 7, 8, 7, 2, 8, 8, 6, 3},
    {3, 1, 11, 5, 2, 9, 7, 3, 10, 6, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 4, 1, 11, 5, 2, 9, 7, 3, 10, 6, 255, 255, 255},
    {4, 0, 1, 2, 1, 11, 2, 11, 7, 2, 3, 10, 6, 255, 255, 255},
    {5, 1, 11, 4, 11, 7, 4, 7, 2, 4, 2, 8, 4, 3, 10, 6},
    {4, 2, 9, 7, 3, 11, 6, 11, 5, 6, 5, 4, 6, 255, 255, 255},
    {5, 0, 8, 5, 8, 6, 5, 6, 3, 5, 3, 11, 5, 2, 9, 7},
    {5, 0, 4, 2, 4, 11, 2, 4, 6, 11, 6, 3, 11, 11, 7, 2},
    {4, 2, 8, 7, 8, 11, 7, 8, 6, 11, 6, 3, 11, 255, 255, 255},
    {3, 3, 10, 7, 10, 8, 7, 8, 9, 7, 255, 255, 255, 255, 255, 255},
    {4, 0, 9, 4, 9, 7, 4, 7, 3, 4, 3, 10, 4, 255, 255, 255},
    {4, 0, 5, 8, 5, 7, 8, 7, 3, 8, 3, 10, 8, 255, 255, 255},
    {3, 3, 10, 7, 10, 4, 7, 4, 5, 7, 255, 255, 255, 255, 255, 255},
    {4, 1, 4, 3, 4, 8, 3, 8, 9, 3, 9, 7, 3, 255, 255, 255},
    {3, 0, 9, 1, 9, 7, 1, 7, 3, 1, 255, 255, 255, 255, 255, 255},
    {5, 0, 5, 8, 5, 7, 8, 7, 3, 8, 3, 1, 8, 1, 4, 8},
    {2, 1, 5, 3, 5, 7, 3, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {4, 1, 11, 5, 3, 10, 7, 10, 8, 7, 8, 9, 7, 255, 255, 255},
    {5, 0, 9, 4, 9, 7, 4, 7, 3, 4, 3, 10, 4, 1, 11, 5},
    {5, 0, 1, 8, 1, 11, 8, 11, 7, 8, 7, 3, 8, 3, 10, 8},
    {4, 1, 11, 4, 11, 7, 4, 7, 3, 4, 3, 10, 4, 255, 255, 255},
    {5, 3, 4, 7, 3, 11, 4, 11, 5, 4, 4, 8, 7, 8, 9, 7},
    {4, 0, 3, 5, 0, 9, 3, 9, 7, 3, 3, 11, 5, 255, 255, 255},
    {2, 0, 4, 8, 3, 11, 7, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 3, 11, 7, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 3, 7, 11, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 8, 4, 3, 7, 11, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 0, 5, 9, 3, 7, 11, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 3, 7, 11, 4, 5, 8, 5, 9, 8, 255, 255, 255, 255, 255, 255},
    {2, 1, 4, 10, 3, 7, 11, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 1, 8, 10, 1, 3, 7, 11, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 9, 1, 4, 10, 3, 7, 11, 255, 255, 255, 255, 255, 255},
    {4, 1, 5, 10, 5, 9, 10, 9, 8, 10, 3, 7, 11, 255, 255, 255},
    {2, 1, 3, 5, 3, 7, 5, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 4, 1, 3, 5, 3, 7, 5, 255, 255, 255, 255, 255, 255},
    {3, 0, 1, 9, 1, 3, 9, 3, 7, 9, 255, 255, 255, 255, 255, 255},
    {4, 1, 3, 4, 3, 7, 4, 7, 9, 4, 9, 8, 4, 255, 255, 255},
    {3, 3, 7, 10, 7, 5, 10, 5, 4, 10, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 5, 8, 10, 5, 10, 3, 5, 3, 7, 5, 255, 255, 255},
    {4, 0, 4, 9, 4, 10, 9, 10, 3, 9, 3, 7, 9, 255, 255, 255},
    {3, 3, 7, 10, 7, 9, 10, 9, 8, 10, 255, 255, 255, 255, 255, 255},
    {2, 2, 6, 8, 3, 7, 11, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 2, 4, 2, 6, 4, 3, 7, 11, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 9, 2, 6, 8, 3, 7, 11, 255, 255, 255, 255, 255, 255},
    {4, 2, 6, 9, 6, 4, 9, 4, 5, 9, 3, 7, 11, 255, 255, 255},
    {3, 1, 4, 10, 2, 6, 8, 3, 7, 11, 255, 255, 255, 255, 255, 255},
    {4, 0, 2, 1, 2, 6, 1, 6, 10, 1, 3, 7, 11, 255, 255, 255},
    {4, 0, 5, 9, 1, 4, 10, 2, 6, 8, 3, 7, 11, 255, 255, 255},
    {5, 1, 5, 10, 5, 9, 10, 9, 2, 10, 2, 6, 10, 3, 7, 11},
    {3, 1, 3, 5, 3, 7, 5, 2, 6, 8, 255, 255, 255, 255, 255, 255},
    {4, 0, 2, 4, 2, 6, 4, 1, 3, 5, 3, 7, 5, 255, 255, 255},
    {4, 0, 1, 9, 1, 3, 9, 3, 7, 9, 2, 6, 8, 255, 255, 255},
    {5, 1, 3, 4, 3, 7, 4, 7, 9, 4, 9, 2, 4, 2, 6, 4},
    {4, 2, 6, 8, 3, 7, 10, 7, 5, 10, 5, 4, 10, 255, 255, 255},
    {5, 0, 2, 5, 2, 6, 5, 6, 10, 5, 10, 3, 5, 3, 7, 5},
    {5, 0, 4, 9, 4, 10, 9, 10, 3, 9, 3, 7, 9, 2, 6, 8},
    {4, 2, 6, 9, 6, 10, 9, 10, 3, 9, 3, 7, 9, 255, 255, 255},
    {2, 2, 9, 3, 9, 11, 3, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 4, 2, 9, 3, 9, 11, 3, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 2, 5, 11, 2, 11, 3, 2, 255, 255, 255, 255, 255, 255},
    {4, 2, 8, 3, 8, 4, 3, 4, 5, 3, 5, 11, 3, 255, 255, 255},
    {3, 1, 4, 10, 2, 9, 3, 9, 11, 3, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 1, 8, 10, 1, 2, 9, 3, 9, 11, 3, 255, 255, 255},
    {4, 0, 5, 2, 5, 11, 2, 11, 3, 2, 1, 4, 10, 255, 255, 255},
    {5, 1, 5, 10, 5, 2, 10, 5, 11, 2, 11, 3, 2, 2, 8, 10},
    {3, 1, 3, 5, 3, 2, 5, 2, 9, 5, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 4, 1, 3, 5, 3, 2, 5, 2, 9, 5, 255, 255, 255},
    {2, 0, 1, 2, 1, 3, 2, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 1, 3, 4, 3, 2, 4, 2, 8, 4, 255, 255, 255, 255, 255, 255},
    {4, 2, 9, 3, 9, 5, 3, 5, 4, 3, 4, 10, 3, 255, 255, 255},
    {5, 0, 8, 5, 8, 10, 5, 10, 3, 5, 3, 2, 5, 2, 9, 5},
    {3, 0, 4, 2, 4, 10, 2, 10, 3, 2, 255, 255, 255, 255, 255, 255},
    {2, 2, 8, 3, 8, 10, 3, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 3, 6, 11, 6, 8, 11, 8, 9, 11, 255, 255, 255, 255, 255, 255},
    {4, 0, 9, 4, 9, 11, 4, 11, 3, 4, 3, 6, 4, 255, 255, 255},
    {4, 0, 5, 8, 5, 11, 8, 11, 3, 8, 3, 6, 8, 255, 255, 255},
    {3, 3, 6, 11, 6, 4, 11, 4, 5, 11, 255, 255, 255, 255, 255, 255},
    {4, 1, 4, 10, 3, 6, 11, 6, 8, 11, 8, 9, 11, 255, 255, 255},
    {5, 0, 9, 1, 9, 6, 1, 9, 11, 6, 11, 3, 6, 6, 10, 1},
    {5, 0, 5, 8, 5, 11, 8, 11, 3, 8, 3, 6, 8, 1, 4, 10},
    {4, 1, 5, 10, 5, 6, 10, 5, 11, 6, 11, 3, 6, 255, 255, 255},
    {4, 1, 3, 5, 3, 6, 5, 6, 8, 5, 8, 9, 5, 255, 255, 255},
    {5, 0, 9, 4, 9, 3, 4, 9, 5, 3, 5, 1, 3, 3, 6, 4},
    {3, 0, 1, 8, 1, 3, 8, 3, 6, 8, 255, 255, 255, 255, 255, 255},
    {2, 1, 3, 4, 3, 6, 4, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {5, 3, 9, 10, 3, 6, 9, 6, 8, 9, 9, 5, 10, 5, 4, 10},
    {2, 0, 9, 5, 3, 6, 10, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {4, 0, 3, 8, 0, 4, 3, 4, 10, 3, 3, 6, 8, 255, 255, 255},
    {1, 3, 6, 10, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 6, 7, 10, 7, 11, 10, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 4, 6, 7, 10, 7, 11, 10, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 9, 6, 7, 10, 7, 11, 10, 255, 255, 255, 255, 255, 255},
    {4, 4, 5, 8, 5, 9, 8, 6, 7, 10, 7, 11, 10, 255, 255, 255},
    {3, 1, 4, 11, 4, 6, 11, 6, 7, 11, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 1, 8, 6, 1, 6, 7, 1, 7, 11, 1, 255, 255, 255},
    {4, 0, 5, 9, 1, 4, 11, 4, 6, 11, 6, 7, 11, 255, 255, 255},
    {5, 1, 8, 11, 1, 5, 8, 5, 9, 8, 8, 6, 11, 6, 7, 11},
    {3, 1, 10, 5, 10, 6, 5, 6, 7, 5, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 4, 1, 10, 5, 10, 6, 5, 6, 7, 5, 255, 255, 255},
    {4, 0, 1, 9, 1, 10, 9, 10, 6, 9, 6, 7, 9, 255, 255, 255},
    {5, 1, 7, 4, 1, 10, 7, 10, 6, 7, 7, 9, 4, 9, 8, 4},
    {2, 4, 6, 5, 6, 7, 5, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 8, 5, 8, 6, 5, 6, 7, 5, 255, 255, 255, 255, 255, 255},
    {3, 0, 4, 9, 4, 6, 9, 6, 7, 9, 255, 255, 255, 255, 255, 255},
    {2, 6, 7, 8, 7, 9, 8, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 2, 7, 8, 7, 11, 8, 11, 10, 8, 255, 255, 255, 255, 255, 255},
    {4, 0, 2, 4, 2, 7, 4, 7, 11, 4, 11, 10, 4, 255, 255, 255},
    {4, 0, 5, 9, 2, 7, 8, 7, 11, 8, 11, 10, 8, 255, 255, 255},
    {5, 2, 10, 9, 2, 7, 10, 7, 11, 10, 10, 4, 9, 4, 5, 9},
    {4, 1, 4, 11, 4, 8, 11, 8, 2, 11, 2, 7, 11, 255, 255, 255},
    {3, 0, 2, 1, 2, 7, 1, 7, 11, 1, 255, 255, 255, 255, 255, 255},
    {5, 0, 5, 9, 1, 4, 11, 4, 8, 11, 8, 2, 11, 2, 7, 11},
    {4, 1, 2, 11, 1, 5, 2, 5, 9, 2, 2, 7, 11, 255, 255, 255},
    {4, 1, 10, 5, 10, 8, 5, 8, 2, 5, 2, 7, 5, 255, 255, 255},
    {5, 0, 2, 4, 2, 7, 4, 7, 10, 4, 7, 5, 10, 5, 1, 10},
    {5, 0, 1, 9, 1, 10, 9, 10, 7, 9, 10, 8, 7, 8, 2, 7},
    {2, 1, 10, 4, 2, 7, 9, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 2, 7, 8, 7, 5, 8, 5, 4, 8, 255, 255, 255, 255, 255, 255},
    {2, 0, 2, 5, 2, 7, 5, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {4, 0, 4, 9, 4, 7, 9, 4, 8, 7, 8, 2, 7, 255, 255, 255},
    {1, 2, 7, 9, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 2, 9, 6, 9, 11, 6, 11, 10, 6, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 4, 2, 9, 6, 9, 11, 6, 11, 10, 6, 255, 255, 255},
    {4, 0, 5, 2, 5, 11, 2, 11, 10, 2, 10, 6, 2, 255, 255, 255},
    {5, 2, 5, 6, 2, 8, 5, 8, 4, 5, 5, 11, 6, 11, 10, 6},
    {4, 1, 4, 11, 4, 6, 11, 6, 2, 11, 2, 9, 11, 255, 255, 255},
    {5, 0, 8, 1, 8, 6, 1, 6, 2, 1, 2, 9, 1, 9, 11, 1},
    {5, 0, 5, 2, 5, 11, 2, 11, 1, 2, 1, 4, 2, 4, 6, 2},
    {2, 1, 5, 11, 2, 8, 6, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {4, 1, 10, 5, 10, 6, 5, 6, 2, 5, 2, 9, 5, 255, 255, 255},
    {5, 0, 8, 4, 1, 10, 5, 10, 6, 5, 6, 2, 5, 2, 9, 5},
    {3, 0, 1, 2, 1, 10, 2, 10, 6, 2, 255, 255, 255, 255, 255, 255},
    {4, 1, 2, 4, 1, 10, 2, 10, 6, 2, 2, 8, 4, 255, 255, 255},
    {3, 2, 9, 6, 9, 5, 6, 5, 4, 6, 255, 255, 255, 255, 255, 255},
    {4, 0, 8, 5, 8, 6, 5, 6, 2, 5, 2, 9, 5, 255, 255, 255},
    {2, 0, 4, 2, 4, 6, 2, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 2, 8, 6, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 8, 9, 10, 9, 11, 10, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 0, 9, 4, 9, 11, 4, 11, 10, 4, 255, 255, 255, 255, 255, 255},
    {3, 0, 5, 8, 5, 11, 8, 11, 10, 8, 255, 255, 255, 255, 255, 255},
    {2, 4, 5, 10, 5, 11, 10, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 1, 4, 11, 4, 8, 11, 8, 9, 11, 255, 255, 255, 255, 255, 255},
    {2, 0, 9, 1, 9, 11, 1, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {4, 0, 5, 8, 5, 11, 8, 11, 1, 8, 1, 4, 8, 255, 255, 255},
    {1, 1, 5, 11, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {3, 1, 10, 5, 10, 8, 5, 8, 9, 5, 255, 255, 255, 255, 255, 255},
    {4, 0, 9, 4, 9, 10, 4, 9, 5, 10, 5, 1, 10, 255, 255, 255},
    {2, 0, 1, 8, 1, 10, 8, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 1, 10, 4, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {2, 4, 8, 5, 8, 9, 5, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 0, 9, 5, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {1, 0, 4, 8, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
    {0, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255},
};

// WEIGHTED: ofdis_fuse_push_weighted -- frame f's observation at pixel o counts with c = p.weight[f * weight_stride
// + o] in place of 1, and only when c is finite and > 0.  The false instance is ofdis_fuse_push.
template <bool WEIGHTED>
__global__ void __launch_bounds__(FUSE_THREADS) fuse_integrate_kernel(FuseGeom g, FuseVolume v, FusePush p) {
  const long long a = (long long)blockIdx.x * FUSE_THREADS + threadIdx.x;
  if (a >= g.count) return;
  const int i = (int)(a % g.nx);
  const long long r = a / g.nx;
  const int j = (int)(r % g.ny), k = (int)(r / g.ny);
  const float X = g.ox + (float)i * g.voxel, Y = g.oy + (float)j * g.voxel, Z = g.oz + (float)k * g.voxel;
  float T = v.T[a], Wt = v.W[a];
  unsigned char c[3] = {0, 0, 0};
  if (v.C) {
    c[0] = v.C[3 * a];
    c[1] = v.C[3 * a + 1];
    c[2] = v.C[3 * a + 2];
  }
  const DispCamera& cam = p.cam;
  for (int f = 0; f < p.n; ++f) {
    const float* q = p.g + 12 * f;
    const float Zc = ((q[8] * X + q[9] * Y) + q[10] * Z) + q[11];
    if (!(Zc > 0.0f)) continue;
    const float Xc = ((q[0] * X + q[1] * Y) + q[2] * Z) + q[3];
    const float Yc = ((q[4] * X + q[5] * Y) + q[6] * Z) + q[7];
    const float uu = ((cam.fx * Xc) / Zc + cam.cx) + 0.5f, vv = ((cam.fy * Yc) / Zc + cam.cy) + 0.5f;
    if (!(uu >= 0.0f && uu < (float)p.w && vv >= 0.0f && vv < (float)p.h)) continue;
    const int px = (int)floorf(uu), py = (int)floorf(vv);
    const size_t o = (size_t)py * p.w + px;
    float cw = 1.0f;
    if constexpr (WEIGHTED) {
      cw = __ldg(p.weight + f * p.weight_stride + o);
      if (!(cw > 0.0f && cw <= FLT_MAX)) continue;
    }
    const float d = __ldg(p.disp + f * p.disp_stride + o);
    const float s = d + cam.doffs;
    if (!known_d(d) || !(s > 0.0f)) continue;
    const float z = cam.fb / s;
    if (z > p.max_depth) continue;
    const float sdf = z - Zc;
    if (sdf < -g.mu) continue;
    const float fv = fminf(1.0f, sdf / g.mu);
    const float W1 = Wt + (WEIGHTED ? cw : 1.0f);
    T = (T * Wt + (WEIGHTED ? fv * cw : fv)) / W1;
    if (v.C) {
      const unsigned char* I = p.frames + f * p.frame_stride + o * p.noc;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float obs = (float)__ldg(I + (p.noc == 3 ? ch : 0));
        c[ch] = (unsigned char)floorf(((float)c[ch] * Wt + (WEIGHTED ? obs * cw : obs)) / W1 + 0.5f);
      }
    }
    Wt = fminf(W1, g.max_weight);
  }
  v.T[a] = T;
  v.W[a] = Wt;
  if (v.C) {
    v.C[3 * a] = c[0];
    v.C[3 * a + 1] = c[1];
    v.C[3 * a + 2] = c[2];
  }
}

// bit e (0 x, 1 y, 2 z): voxel a = (i, j, k) and its neighbour along e form a crossing
__device__ __forceinline__ unsigned crossings(const FuseGeom& g, const FuseVolume& v, float minw, long long a) {
  if (a >= g.count) return 0u;
  const float Ta = v.T[a], Wa = v.W[a];
  if (!(Wa >= minw && fabsf(Ta) < 1.0f)) return 0u;
  const int i = (int)(a % g.nx);
  const long long r = a / g.nx;
  const int j = (int)(r % g.ny), k = (int)(r / g.ny);
  const bool in[3] = {i + 1 < g.nx, j + 1 < g.ny, k + 1 < g.nz};
  const long long step[3] = {1, g.nx, (long long)g.nx * g.ny};
  unsigned m = 0;
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    if (!in[e]) continue;
    const float Tb = v.T[a + step[e]], Wb = v.W[a + step[e]];
    if (Wb >= minw && fabsf(Tb) < 1.0f && ((Ta > 0.0f) != (Tb > 0.0f))) m |= 1u << e;
  }
  return m;
}

__global__ void __launch_bounds__(FUSE_THREADS) fuse_count_kernel(FuseGeom g, FuseVolume v, float minw,
                                                                  unsigned long long* bsum) {
  __shared__ unsigned int sw[FUSE_THREADS / 32];
  const long long a0 = (long long)blockIdx.x * FUSE_BLOCK + (long long)threadIdx.x * FUSE_VPT;
  unsigned cnt = 0;
#pragma unroll
  for (int q = 0; q < FUSE_VPT; ++q) cnt += __popc(crossings(g, v, minw, a0 + q));
  unsigned int total;
  block_exclusive_scan<FUSE_THREADS>(cnt, sw, total);
  if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

// exclusive 64-bit scan of the nb block counts in place; the sum to *total
__global__ void __launch_bounds__(FUSE_SCAN_THREADS) fuse_scan_kernel(unsigned long long* bsum, int nb,
                                                                      unsigned long long* total) {
  __shared__ unsigned long long sw[FUSE_SCAN_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long carry = 0;
  for (int base = 0; base < nb; base += FUSE_SCAN_THREADS) {
    const int idx = base + threadIdx.x;
    const unsigned long long val = idx < nb ? bsum[idx] : 0ull;
    unsigned long long x = val;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) sw[warp] = x;
    __syncthreads();
    if (warp == 0) {
      unsigned long long s = sw[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += y;
      }
      sw[lane] = s;
    }
    __syncthreads();
    if (idx < nb) bsum[idx] = carry + x - val + (warp ? sw[warp - 1] : 0ull);
    carry += sw[FUSE_SCAN_THREADS / 32 - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

// BASES: also vbase[a] = the index of voxel a's first crossing, for every voxel with a crossing, whatever the capacity
template <bool BASES>
__global__ void __launch_bounds__(FUSE_THREADS) fuse_write_kernel(FuseGeom g, FuseVolume v, float minw,
                                                                  const unsigned long long* bsum,
                                                                  ofdis_fuse_point* out, long long cap,
                                                                  unsigned int* vbase) {
  __shared__ unsigned int sw[FUSE_THREADS / 32];
  const long long a0 = (long long)blockIdx.x * FUSE_BLOCK + (long long)threadIdx.x * FUSE_VPT;
  unsigned m[FUSE_VPT], cnt = 0;
#pragma unroll
  for (int q = 0; q < FUSE_VPT; ++q) {
    m[q] = crossings(g, v, minw, a0 + q);
    cnt += __popc(m[q]);
  }
  unsigned int total;
  const unsigned int ex = block_exclusive_scan<FUSE_THREADS>(cnt, sw, total);
  unsigned long long o = bsum[blockIdx.x] + ex;
  if (BASES) {
    unsigned long long ob = o;
#pragma unroll
    for (int q = 0; q < FUSE_VPT; ++q) {
      if (m[q]) vbase[a0 + q] = (unsigned int)ob;
      ob += __popc(m[q]);
    }
  }
  if (!cnt || o >= (unsigned long long)cap) return;
#pragma unroll
  for (int q = 0; q < FUSE_VPT; ++q) {
    if (!m[q]) continue;
    const long long a = a0 + q;
    const int i = (int)(a % g.nx);
    const long long r = a / g.nx;
    const int j = (int)(r % g.ny), k = (int)(r / g.ny);
    const long long sy = g.nx, sz = (long long)g.nx * g.ny;
    const float* T = v.T;
    const float Ta = T[a];
    const float gx = T[a - i + min(i + 1, g.nx - 1)] - T[a - i + max(i - 1, 0)];
    const float gy = T[a + (min(j + 1, g.ny - 1) - j) * sy] - T[a + (max(j - 1, 0) - j) * sy];
    const float gz = T[a + (min(k + 1, g.nz - 1) - k) * sz] - T[a + (max(k - 1, 0) - k) * sz];
    const float L = sqrtf((gx * gx + gy * gy) + gz * gz);
    const float nrm[3] = {L > 0.0f ? gx / L : qnan(), L > 0.0f ? gy / L : qnan(), L > 0.0f ? gz / L : qnan()};
    const float P[3] = {g.ox + (float)i * g.voxel, g.oy + (float)j * g.voxel, g.oz + (float)k * g.voxel};
    const long long step[3] = {1, sy, sz};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      if (!((m[q] >> e) & 1u)) continue;
      if (o >= (unsigned long long)cap) return;
      const long long b = a + step[e];
      const float Tb = T[b];
      const float t = Ta / (Ta - Tb);
      const float dt = t * g.voxel;
      ofdis_fuse_point rec;
      rec.x = e == 0 ? P[0] + dt : P[0];
      rec.y = e == 1 ? P[1] + dt : P[1];
      rec.z = e == 2 ? P[2] + dt : P[2];
      rec.nx = nrm[0];
      rec.ny = nrm[1];
      rec.nz = nrm[2];
      const long long src = t < 0.5f ? a : b;
      rec.r = v.C ? v.C[3 * src] : 0;
      rec.g = v.C ? v.C[3 * src + 1] : 0;
      rec.b = v.C ? v.C[3 * src + 2] : 0;
      rec.pad = 0;
      out[o++] = rec;
    }
  }
}

// the case of the cube whose corner 0 is voxel a, or -1 where the cube does not exist or is not meshed (a corner fails
// W >= minw && fabsf(T) < 1)
__device__ __forceinline__ int cube_case(const FuseGeom& g, const FuseVolume& v, float minw, long long a) {
  if (a >= g.count) return -1;
  const int i = (int)(a % g.nx);
  const long long r = a / g.nx;
  const int j = (int)(r % g.ny), k = (int)(r / g.ny);
  if (i + 1 >= g.nx || j + 1 >= g.ny || k + 1 >= g.nz) return -1;
  const long long sy = g.nx, sz = (long long)g.nx * g.ny;
  int c = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const long long b = a + (q & 1) + ((q >> 1) & 1) * sy + (q >> 2) * sz;
    const float T = __ldg(v.T + b), W = __ldg(v.W + b);
    if (!(W >= minw && fabsf(T) < 1.0f)) return -1;
    c |= (T > 0.0f ? 1 : 0) << q;
  }
  return c;
}

__global__ void __launch_bounds__(FUSE_THREADS) fuse_cube_count_kernel(FuseGeom g, FuseVolume v, float minw,
                                                                       unsigned long long* bsum) {
  __shared__ unsigned int sw[FUSE_THREADS / 32];
  const long long a0 = (long long)blockIdx.x * FUSE_BLOCK + (long long)threadIdx.x * FUSE_VPT;
  unsigned cnt = 0;
#pragma unroll
  for (int q = 0; q < FUSE_VPT; ++q) {
    const int c = cube_case(g, v, minw, a0 + q);
    if (c >= 0) cnt += FUSE_MC[c][0];
  }
  unsigned int total;
  block_exclusive_scan<FUSE_THREADS>(cnt, sw, total);
  if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

// the vertex of cube edge n (lower corner q, axis e) of the cube at voxel a: the first vertex of corner q's voxel plus
// that voxel's crossings along the axes before e
__device__ __forceinline__ unsigned int edge_vertex(const FuseGeom& g, const FuseVolume& v, float minw,
                                                    const unsigned int* vbase, long long a, int n) {
  const int e = n >> 2, r = n & 3;
  const int q = (r & ((1 << e) - 1)) | ((r >> e) << (e + 1));
  const long long b = a + (q & 1) + ((q >> 1) & 1) * (long long)g.nx + (q >> 2) * ((long long)g.nx * g.ny);
  return vbase[b] + (unsigned int)__popc(crossings(g, v, minw, b) & ((1u << e) - 1u));
}

__global__ void __launch_bounds__(FUSE_THREADS) fuse_face_kernel(FuseGeom g, FuseVolume v, float minw,
                                                                 const unsigned long long* bsum,
                                                                 const unsigned int* vbase, unsigned int* faces,
                                                                 long long cap) {
  __shared__ unsigned int sw[FUSE_THREADS / 32];
  const long long a0 = (long long)blockIdx.x * FUSE_BLOCK + (long long)threadIdx.x * FUSE_VPT;
  int c[FUSE_VPT];
  unsigned cnt = 0;
#pragma unroll
  for (int q = 0; q < FUSE_VPT; ++q) {
    c[q] = cube_case(g, v, minw, a0 + q);
    if (c[q] >= 0) cnt += FUSE_MC[c[q]][0];
  }
  unsigned int total;
  const unsigned int ex = block_exclusive_scan<FUSE_THREADS>(cnt, sw, total);
  unsigned long long o = bsum[blockIdx.x] + ex;
  if (!cnt || o >= (unsigned long long)cap) return;
#pragma unroll
  for (int q = 0; q < FUSE_VPT; ++q) {
    if (c[q] < 0) continue;
    const int nt = FUSE_MC[c[q]][0];
    for (int t = 0; t < nt; ++t) {
      if (o >= (unsigned long long)cap) return;
      unsigned int* f = faces + 3 * o;
#pragma unroll
      for (int s = 0; s < 3; ++s) f[s] = edge_vertex(g, v, minw, vbase, a0 + q, FUSE_MC[c[q]][1 + 3 * t + s]);
      ++o;
    }
  }
}

// trilinear T at voxel coordinates q, or false where a corner lies outside or has W < minw
__device__ __forceinline__ bool fuse_sample(const FuseGeom& g, const FuseVolume& v, float minw, const float (&q)[3],
                                            float& out) {
  const int n[3] = {g.nx, g.ny, g.nz};
  int i0[3];
  float fr[3];
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    const float fl = floorf(q[e]);
    if (!(fl >= 0.0f && fl <= (float)(n[e] - 2))) return false;
    i0[e] = (int)fl;
    fr[e] = q[e] - fl;
  }
  const long long sy = g.nx, sz = (long long)g.nx * g.ny;
  const long long base = ((long long)i0[2] * g.ny + i0[1]) * g.nx + i0[0];
  const long long off[8] = {0, 1, sy, sy + 1, sz, sz + 1, sz + sy, sz + sy + 1};
  float c[8];
#pragma unroll
  for (int q8 = 0; q8 < 8; ++q8)
    if (!(__ldg(v.W + base + off[q8]) >= minw)) return false;
#pragma unroll
  for (int q8 = 0; q8 < 8; ++q8) c[q8] = __ldg(v.T + base + off[q8]);
  const float gx = 1.0f - fr[0], gy = 1.0f - fr[1], gz = 1.0f - fr[2];
  const float x00 = c[0] * gx + c[1] * fr[0], x10 = c[2] * gx + c[3] * fr[0];
  const float x01 = c[4] * gx + c[5] * fr[0], x11 = c[6] * gx + c[7] * fr[0];
  const float y0 = x00 * gy + x10 * fr[1], y1 = x01 * gy + x11 * fr[1];
  out = y0 * gz + y1 * fr[2];
  return true;
}

__global__ void __launch_bounds__(32 * FUSE_RENDER_ROWS) fuse_render_kernel(FuseGeom g, FuseVolume v, FuseRender p) {
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * FUSE_RENDER_ROWS + threadIdx.y, k = blockIdx.z;
  if (x >= p.w || y >= p.h) return;
  const float* P = p.pose + 12 * k;
  const DispCamera& cam = p.cam;
  const float r0 = ((float)x - cam.cx) / cam.fx, r1 = ((float)y - cam.cy) / cam.fy;
  float depth = qnan();
  bool prev = false;
  float Tp = 0.0f, Zp = 0.0f;
  for (int s = 0; s <= FUSE_MAX_SAMPLES; ++s) {
    const float Zs = p.z_near + (float)s * p.step;
    if (!(Zs <= p.z_far)) break;
    const float cx = r0 * Zs, cy = r1 * Zs;
    float q[3];
    q[0] = ((((P[0] * cx + P[1] * cy) + P[2] * Zs) + P[3]) - g.ox) / g.voxel;
    q[1] = ((((P[4] * cx + P[5] * cy) + P[6] * Zs) + P[7]) - g.oy) / g.voxel;
    q[2] = ((((P[8] * cx + P[9] * cy) + P[10] * Zs) + P[11]) - g.oz) / g.voxel;
    float T;
    const bool known = fuse_sample(g, v, p.min_weight, q, T);
    if (known && prev && Tp > 0.0f && T <= 0.0f) {
      depth = Zp + p.step * (Tp / (Tp - T));
      break;
    }
    prev = known;
    Tp = T;
    Zp = Zs;
  }
  p.depth[((size_t)k * p.h + y) * p.w + x] = depth;
}

}  // namespace

int launch_fuse_push(const FuseGeom& g, const FuseVolume& v, const FusePush& p, cudaStream_t st) {
  const long long blocks = (g.count + FUSE_THREADS - 1) / FUSE_THREADS;
  if (p.weight) fuse_integrate_kernel<true><<<(unsigned)blocks, FUSE_THREADS, 0, st>>>(g, v, p);
  else fuse_integrate_kernel<false><<<(unsigned)blocks, FUSE_THREADS, 0, st>>>(g, v, p);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_fuse_count(const FuseGeom& g, const FuseVolume& v, float min_weight, const FuseWork& ws, cudaStream_t st) {
  const int nb = (int)((g.count + FUSE_BLOCK - 1) / FUSE_BLOCK);
  fuse_count_kernel<<<nb, FUSE_THREADS, 0, st>>>(g, v, min_weight, ws.bsum);
  fuse_scan_kernel<<<1, FUSE_SCAN_THREADS, 0, st>>>(ws.bsum, nb, ws.total);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

int launch_fuse_write(const FuseGeom& g, const FuseVolume& v, float min_weight, const FuseWork& ws,
                      ofdis_fuse_point* out, long long cap, cudaStream_t st, unsigned int* vbase) {
  const int nb = (int)((g.count + FUSE_BLOCK - 1) / FUSE_BLOCK);
  if (vbase)
    fuse_write_kernel<true><<<nb, FUSE_THREADS, 0, st>>>(g, v, min_weight, ws.bsum, out, cap, vbase);
  else
    fuse_write_kernel<false><<<nb, FUSE_THREADS, 0, st>>>(g, v, min_weight, ws.bsum, out, cap, nullptr);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_fuse_cube_count(const FuseGeom& g, const FuseVolume& v, float min_weight, const FuseMeshWork& mw,
                           cudaStream_t st) {
  const int nb = (int)((g.count + FUSE_BLOCK - 1) / FUSE_BLOCK);
  fuse_cube_count_kernel<<<nb, FUSE_THREADS, 0, st>>>(g, v, min_weight, mw.bsum);
  fuse_scan_kernel<<<1, FUSE_SCAN_THREADS, 0, st>>>(mw.bsum, nb, mw.total);
  return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

int launch_fuse_faces(const FuseGeom& g, const FuseVolume& v, float min_weight, const FuseMeshWork& mw,
                      unsigned int* faces, long long cap, cudaStream_t st) {
  const int nb = (int)((g.count + FUSE_BLOCK - 1) / FUSE_BLOCK);
  fuse_face_kernel<<<nb, FUSE_THREADS, 0, st>>>(g, v, min_weight, mw.bsum, mw.vbase, faces, cap);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_fuse_render(const FuseGeom& g, const FuseVolume& v, const FuseRender& p, int n, cudaStream_t st) {
  const dim3 block(32, FUSE_RENDER_ROWS), grid((p.w + 31) / 32, (p.h + FUSE_RENDER_ROWS - 1) / FUSE_RENDER_ROWS, n);
  fuse_render_kernel<<<grid, block, 0, st>>>(g, v, p);
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace ofdis
