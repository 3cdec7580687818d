// mesh.cu -- mesh export (NeRFRenderer.export_mesh, nerf/renderer.py:157-330): marching cubes over the density volume and the
// texel pass of a closed-form per-face texture atlas.  Compiled with -fmad=false: vertex interpolation and the texel -> xyz map are
// single-rounding fp32 so oracle/mesh_ref.py reproduces them bit for bit.
//
// Marching cubes (Lorensen & Cline 1987) with the public-domain 256-case triangle table of Paul Bourke / Cory Bloyd:
//   * volume fp32 [nx, ny, nz], C order, (i, j, k) <-> (x, y, z).  A corner is inside iff sigma > iso; bit m of the cube index is set
//     iff corner m (Bourke numbering, c_corner below) is not inside.
//   * one vertex per crossing grid edge, owned by its lower end point p: p + t e_a, t = (iso - s_p) / (s_{p+e_a} - s_p).
//     Numbering: grid points in C order, then axis x < y < z.
//   * faces: cells in C order, triangles in table order.  As written, the table winds each triangle so that its right-hand normal
//     points to the corners with sigma <= iso (out of the solid), which is the orientation wanted: triangles are emitted unchanged.
//   * pipeline: k_mc_count (per point: owned crossings, cell triangle count; block scan + decoupled look-back over ticketed blocks,
//     so vertex / face offsets are ordered by point index and no atomic decides any order) -> the caller reads (V, F) ->
//     k_mc_emit (every point writes its vertices and its cell's triangles at the offsets the count pass stored).
#include "mi3d_common.cuh"
#include "../../include/mi3d.h"

namespace {

constexpr int kMcThreads = 256;

__constant__ int8_t c_corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
// edge e runs from corner c_edge_from[e] along +axis c_edge_axis[e]
__constant__ int8_t c_edge_from[12] = {0, 1, 3, 0, 4, 5, 7, 4, 0, 1, 2, 3};
__constant__ int8_t c_edge_axis[12] = {0, 1, 0, 1, 0, 1, 0, 1, 2, 2, 2, 2};

__constant__ int8_t c_tri[256][16] = {
    {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 8, 3, 9, 8, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 1, 2, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 2, 10, 0, 2, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 8, 3, 2, 10, 8, 10, 9, 8, -1, -1, -1, -1, -1, -1, -1},
    {3, 11, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 11, 2, 8, 11, 0, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 9, 0, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 11, 2, 1, 9, 11, 9, 8, 11, -1, -1, -1, -1, -1, -1, -1},
    {3, 10, 1, 11, 10, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 10, 1, 0, 8, 10, 8, 11, 10, -1, -1, -1, -1, -1, -1, -1},
    {3, 9, 0, 3, 11, 9, 11, 10, 9, -1, -1, -1, -1, -1, -1, -1},
    {9, 8, 10, 10, 8, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 7, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 3, 0, 7, 3, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 9, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 1, 9, 4, 7, 1, 7, 3, 1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 4, 7, 3, 0, 4, 1, 2, 10, -1, -1, -1, -1, -1, -1, -1},
    {9, 2, 10, 9, 0, 2, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1},
    {2, 10, 9, 2, 9, 7, 2, 7, 3, 7, 9, 4, -1, -1, -1, -1},
    {8, 4, 7, 3, 11, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {11, 4, 7, 11, 2, 4, 2, 0, 4, -1, -1, -1, -1, -1, -1, -1},
    {9, 0, 1, 8, 4, 7, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1},
    {4, 7, 11, 9, 4, 11, 9, 11, 2, 9, 2, 1, -1, -1, -1, -1},
    {3, 10, 1, 3, 11, 10, 7, 8, 4, -1, -1, -1, -1, -1, -1, -1},
    {1, 11, 10, 1, 4, 11, 1, 0, 4, 7, 11, 4, -1, -1, -1, -1},
    {4, 7, 8, 9, 0, 11, 9, 11, 10, 11, 0, 3, -1, -1, -1, -1},
    {4, 7, 11, 4, 11, 9, 9, 11, 10, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 4, 0, 8, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 5, 4, 1, 5, 0, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 5, 4, 8, 3, 5, 3, 1, 5, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 9, 5, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 8, 1, 2, 10, 4, 9, 5, -1, -1, -1, -1, -1, -1, -1},
    {5, 2, 10, 5, 4, 2, 4, 0, 2, -1, -1, -1, -1, -1, -1, -1},
    {2, 10, 5, 3, 2, 5, 3, 5, 4, 3, 4, 8, -1, -1, -1, -1},
    {9, 5, 4, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 11, 2, 0, 8, 11, 4, 9, 5, -1, -1, -1, -1, -1, -1, -1},
    {0, 5, 4, 0, 1, 5, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1},
    {2, 1, 5, 2, 5, 8, 2, 8, 11, 4, 8, 5, -1, -1, -1, -1},
    {10, 3, 11, 10, 1, 3, 9, 5, 4, -1, -1, -1, -1, -1, -1, -1},
    {4, 9, 5, 0, 8, 1, 8, 10, 1, 8, 11, 10, -1, -1, -1, -1},
    {5, 4, 0, 5, 0, 11, 5, 11, 10, 11, 0, 3, -1, -1, -1, -1},
    {5, 4, 8, 5, 8, 10, 10, 8, 11, -1, -1, -1, -1, -1, -1, -1},
    {9, 7, 8, 5, 7, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 3, 0, 9, 5, 3, 5, 7, 3, -1, -1, -1, -1, -1, -1, -1},
    {0, 7, 8, 0, 1, 7, 1, 5, 7, -1, -1, -1, -1, -1, -1, -1},
    {1, 5, 3, 3, 5, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 7, 8, 9, 5, 7, 10, 1, 2, -1, -1, -1, -1, -1, -1, -1},
    {10, 1, 2, 9, 5, 0, 5, 3, 0, 5, 7, 3, -1, -1, -1, -1},
    {8, 0, 2, 8, 2, 5, 8, 5, 7, 10, 5, 2, -1, -1, -1, -1},
    {2, 10, 5, 2, 5, 3, 3, 5, 7, -1, -1, -1, -1, -1, -1, -1},
    {7, 9, 5, 7, 8, 9, 3, 11, 2, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 7, 9, 7, 2, 9, 2, 0, 2, 7, 11, -1, -1, -1, -1},
    {2, 3, 11, 0, 1, 8, 1, 7, 8, 1, 5, 7, -1, -1, -1, -1},
    {11, 2, 1, 11, 1, 7, 7, 1, 5, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 8, 8, 5, 7, 10, 1, 3, 10, 3, 11, -1, -1, -1, -1},
    {5, 7, 0, 5, 0, 9, 7, 11, 0, 1, 0, 10, 11, 10, 0, -1},
    {11, 10, 0, 11, 0, 3, 10, 5, 0, 8, 0, 7, 5, 7, 0, -1},
    {11, 10, 5, 7, 11, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {10, 6, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 0, 1, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 8, 3, 1, 9, 8, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1},
    {1, 6, 5, 2, 6, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 6, 5, 1, 2, 6, 3, 0, 8, -1, -1, -1, -1, -1, -1, -1},
    {9, 6, 5, 9, 0, 6, 0, 2, 6, -1, -1, -1, -1, -1, -1, -1},
    {5, 9, 8, 5, 8, 2, 5, 2, 6, 3, 2, 8, -1, -1, -1, -1},
    {2, 3, 11, 10, 6, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {11, 0, 8, 11, 2, 0, 10, 6, 5, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 9, 2, 3, 11, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1},
    {5, 10, 6, 1, 9, 2, 9, 11, 2, 9, 8, 11, -1, -1, -1, -1},
    {6, 3, 11, 6, 5, 3, 5, 1, 3, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 11, 0, 11, 5, 0, 5, 1, 5, 11, 6, -1, -1, -1, -1},
    {3, 11, 6, 0, 3, 6, 0, 6, 5, 0, 5, 9, -1, -1, -1, -1},
    {6, 5, 9, 6, 9, 11, 11, 9, 8, -1, -1, -1, -1, -1, -1, -1},
    {5, 10, 6, 4, 7, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 3, 0, 4, 7, 3, 6, 5, 10, -1, -1, -1, -1, -1, -1, -1},
    {1, 9, 0, 5, 10, 6, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1},
    {10, 6, 5, 1, 9, 7, 1, 7, 3, 7, 9, 4, -1, -1, -1, -1},
    {6, 1, 2, 6, 5, 1, 4, 7, 8, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 5, 5, 2, 6, 3, 0, 4, 3, 4, 7, -1, -1, -1, -1},
    {8, 4, 7, 9, 0, 5, 0, 6, 5, 0, 2, 6, -1, -1, -1, -1},
    {7, 3, 9, 7, 9, 4, 3, 2, 9, 5, 9, 6, 2, 6, 9, -1},
    {3, 11, 2, 7, 8, 4, 10, 6, 5, -1, -1, -1, -1, -1, -1, -1},
    {5, 10, 6, 4, 7, 2, 4, 2, 0, 2, 7, 11, -1, -1, -1, -1},
    {0, 1, 9, 4, 7, 8, 2, 3, 11, 5, 10, 6, -1, -1, -1, -1},
    {9, 2, 1, 9, 11, 2, 9, 4, 11, 7, 11, 4, 5, 10, 6, -1},
    {8, 4, 7, 3, 11, 5, 3, 5, 1, 5, 11, 6, -1, -1, -1, -1},
    {5, 1, 11, 5, 11, 6, 1, 0, 11, 7, 11, 4, 0, 4, 11, -1},
    {0, 5, 9, 0, 6, 5, 0, 3, 6, 11, 6, 3, 8, 4, 7, -1},
    {6, 5, 9, 6, 9, 11, 4, 7, 9, 7, 11, 9, -1, -1, -1, -1},
    {10, 4, 9, 6, 4, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 10, 6, 4, 9, 10, 0, 8, 3, -1, -1, -1, -1, -1, -1, -1},
    {10, 0, 1, 10, 6, 0, 6, 4, 0, -1, -1, -1, -1, -1, -1, -1},
    {8, 3, 1, 8, 1, 6, 8, 6, 4, 6, 1, 10, -1, -1, -1, -1},
    {1, 4, 9, 1, 2, 4, 2, 6, 4, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 8, 1, 2, 9, 2, 4, 9, 2, 6, 4, -1, -1, -1, -1},
    {0, 2, 4, 4, 2, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 3, 2, 8, 2, 4, 4, 2, 6, -1, -1, -1, -1, -1, -1, -1},
    {10, 4, 9, 10, 6, 4, 11, 2, 3, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 2, 2, 8, 11, 4, 9, 10, 4, 10, 6, -1, -1, -1, -1},
    {3, 11, 2, 0, 1, 6, 0, 6, 4, 6, 1, 10, -1, -1, -1, -1},
    {6, 4, 1, 6, 1, 10, 4, 8, 1, 2, 1, 11, 8, 11, 1, -1},
    {9, 6, 4, 9, 3, 6, 9, 1, 3, 11, 6, 3, -1, -1, -1, -1},
    {8, 11, 1, 8, 1, 0, 11, 6, 1, 9, 1, 4, 6, 4, 1, -1},
    {3, 11, 6, 3, 6, 0, 0, 6, 4, -1, -1, -1, -1, -1, -1, -1},
    {6, 4, 8, 11, 6, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {7, 10, 6, 7, 8, 10, 8, 9, 10, -1, -1, -1, -1, -1, -1, -1},
    {0, 7, 3, 0, 10, 7, 0, 9, 10, 6, 7, 10, -1, -1, -1, -1},
    {10, 6, 7, 1, 10, 7, 1, 7, 8, 1, 8, 0, -1, -1, -1, -1},
    {10, 6, 7, 10, 7, 1, 1, 7, 3, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 6, 1, 6, 8, 1, 8, 9, 8, 6, 7, -1, -1, -1, -1},
    {2, 6, 9, 2, 9, 1, 6, 7, 9, 0, 9, 3, 7, 3, 9, -1},
    {7, 8, 0, 7, 0, 6, 6, 0, 2, -1, -1, -1, -1, -1, -1, -1},
    {7, 3, 2, 6, 7, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 3, 11, 10, 6, 8, 10, 8, 9, 8, 6, 7, -1, -1, -1, -1},
    {2, 0, 7, 2, 7, 11, 0, 9, 7, 6, 7, 10, 9, 10, 7, -1},
    {1, 8, 0, 1, 7, 8, 1, 10, 7, 6, 7, 10, 2, 3, 11, -1},
    {11, 2, 1, 11, 1, 7, 10, 6, 1, 6, 7, 1, -1, -1, -1, -1},
    {8, 9, 6, 8, 6, 7, 9, 1, 6, 11, 6, 3, 1, 3, 6, -1},
    {0, 9, 1, 11, 6, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {7, 8, 0, 7, 0, 6, 3, 11, 0, 11, 6, 0, -1, -1, -1, -1},
    {7, 11, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {7, 6, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 8, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 9, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 1, 9, 8, 3, 1, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1},
    {10, 1, 2, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 3, 0, 8, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1},
    {2, 9, 0, 2, 10, 9, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1},
    {6, 11, 7, 2, 10, 3, 10, 8, 3, 10, 9, 8, -1, -1, -1, -1},
    {7, 2, 3, 6, 2, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {7, 0, 8, 7, 6, 0, 6, 2, 0, -1, -1, -1, -1, -1, -1, -1},
    {2, 7, 6, 2, 3, 7, 0, 1, 9, -1, -1, -1, -1, -1, -1, -1},
    {1, 6, 2, 1, 8, 6, 1, 9, 8, 8, 7, 6, -1, -1, -1, -1},
    {10, 7, 6, 10, 1, 7, 1, 3, 7, -1, -1, -1, -1, -1, -1, -1},
    {10, 7, 6, 1, 7, 10, 1, 8, 7, 1, 0, 8, -1, -1, -1, -1},
    {0, 3, 7, 0, 7, 10, 0, 10, 9, 6, 10, 7, -1, -1, -1, -1},
    {7, 6, 10, 7, 10, 8, 8, 10, 9, -1, -1, -1, -1, -1, -1, -1},
    {6, 8, 4, 11, 8, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 6, 11, 3, 0, 6, 0, 4, 6, -1, -1, -1, -1, -1, -1, -1},
    {8, 6, 11, 8, 4, 6, 9, 0, 1, -1, -1, -1, -1, -1, -1, -1},
    {9, 4, 6, 9, 6, 3, 9, 3, 1, 11, 3, 6, -1, -1, -1, -1},
    {6, 8, 4, 6, 11, 8, 2, 10, 1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 3, 0, 11, 0, 6, 11, 0, 4, 6, -1, -1, -1, -1},
    {4, 11, 8, 4, 6, 11, 0, 2, 9, 2, 10, 9, -1, -1, -1, -1},
    {10, 9, 3, 10, 3, 2, 9, 4, 3, 11, 3, 6, 4, 6, 3, -1},
    {8, 2, 3, 8, 4, 2, 4, 6, 2, -1, -1, -1, -1, -1, -1, -1},
    {0, 4, 2, 4, 6, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 9, 0, 2, 3, 4, 2, 4, 6, 4, 3, 8, -1, -1, -1, -1},
    {1, 9, 4, 1, 4, 2, 2, 4, 6, -1, -1, -1, -1, -1, -1, -1},
    {8, 1, 3, 8, 6, 1, 8, 4, 6, 6, 10, 1, -1, -1, -1, -1},
    {10, 1, 0, 10, 0, 6, 6, 0, 4, -1, -1, -1, -1, -1, -1, -1},
    {4, 6, 3, 4, 3, 8, 6, 10, 3, 0, 3, 9, 10, 9, 3, -1},
    {10, 9, 4, 6, 10, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 9, 5, 7, 6, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 4, 9, 5, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1},
    {5, 0, 1, 5, 4, 0, 7, 6, 11, -1, -1, -1, -1, -1, -1, -1},
    {11, 7, 6, 8, 3, 4, 3, 5, 4, 3, 1, 5, -1, -1, -1, -1},
    {9, 5, 4, 10, 1, 2, 7, 6, 11, -1, -1, -1, -1, -1, -1, -1},
    {6, 11, 7, 1, 2, 10, 0, 8, 3, 4, 9, 5, -1, -1, -1, -1},
    {7, 6, 11, 5, 4, 10, 4, 2, 10, 4, 0, 2, -1, -1, -1, -1},
    {3, 4, 8, 3, 5, 4, 3, 2, 5, 10, 5, 2, 11, 7, 6, -1},
    {7, 2, 3, 7, 6, 2, 5, 4, 9, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 4, 0, 8, 6, 0, 6, 2, 6, 8, 7, -1, -1, -1, -1},
    {3, 6, 2, 3, 7, 6, 1, 5, 0, 5, 4, 0, -1, -1, -1, -1},
    {6, 2, 8, 6, 8, 7, 2, 1, 8, 4, 8, 5, 1, 5, 8, -1},
    {9, 5, 4, 10, 1, 6, 1, 7, 6, 1, 3, 7, -1, -1, -1, -1},
    {1, 6, 10, 1, 7, 6, 1, 0, 7, 8, 7, 0, 9, 5, 4, -1},
    {4, 0, 10, 4, 10, 5, 0, 3, 10, 6, 10, 7, 3, 7, 10, -1},
    {7, 6, 10, 7, 10, 8, 5, 4, 10, 4, 8, 10, -1, -1, -1, -1},
    {6, 9, 5, 6, 11, 9, 11, 8, 9, -1, -1, -1, -1, -1, -1, -1},
    {3, 6, 11, 0, 6, 3, 0, 5, 6, 0, 9, 5, -1, -1, -1, -1},
    {0, 11, 8, 0, 5, 11, 0, 1, 5, 5, 6, 11, -1, -1, -1, -1},
    {6, 11, 3, 6, 3, 5, 5, 3, 1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 9, 5, 11, 9, 11, 8, 11, 5, 6, -1, -1, -1, -1},
    {0, 11, 3, 0, 6, 11, 0, 9, 6, 5, 6, 9, 1, 2, 10, -1},
    {11, 8, 5, 11, 5, 6, 8, 0, 5, 10, 5, 2, 0, 2, 5, -1},
    {6, 11, 3, 6, 3, 5, 2, 10, 3, 10, 5, 3, -1, -1, -1, -1},
    {5, 8, 9, 5, 2, 8, 5, 6, 2, 3, 8, 2, -1, -1, -1, -1},
    {9, 5, 6, 9, 6, 0, 0, 6, 2, -1, -1, -1, -1, -1, -1, -1},
    {1, 5, 8, 1, 8, 0, 5, 6, 8, 3, 8, 2, 6, 2, 8, -1},
    {1, 5, 6, 2, 1, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 3, 6, 1, 6, 10, 3, 8, 6, 5, 6, 9, 8, 9, 6, -1},
    {10, 1, 0, 10, 0, 6, 9, 5, 0, 5, 6, 0, -1, -1, -1, -1},
    {0, 3, 8, 5, 6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {10, 5, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {11, 5, 10, 7, 5, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {11, 5, 10, 11, 7, 5, 8, 3, 0, -1, -1, -1, -1, -1, -1, -1},
    {5, 11, 7, 5, 10, 11, 1, 9, 0, -1, -1, -1, -1, -1, -1, -1},
    {10, 7, 5, 10, 11, 7, 9, 8, 1, 8, 3, 1, -1, -1, -1, -1},
    {11, 1, 2, 11, 7, 1, 7, 5, 1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 1, 2, 7, 1, 7, 5, 7, 2, 11, -1, -1, -1, -1},
    {9, 7, 5, 9, 2, 7, 9, 0, 2, 2, 11, 7, -1, -1, -1, -1},
    {7, 5, 2, 7, 2, 11, 5, 9, 2, 3, 2, 8, 9, 8, 2, -1},
    {2, 5, 10, 2, 3, 5, 3, 7, 5, -1, -1, -1, -1, -1, -1, -1},
    {8, 2, 0, 8, 5, 2, 8, 7, 5, 10, 2, 5, -1, -1, -1, -1},
    {9, 0, 1, 5, 10, 3, 5, 3, 7, 3, 10, 2, -1, -1, -1, -1},
    {9, 8, 2, 9, 2, 1, 8, 7, 2, 10, 2, 5, 7, 5, 2, -1},
    {1, 3, 5, 3, 7, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 7, 0, 7, 1, 1, 7, 5, -1, -1, -1, -1, -1, -1, -1},
    {9, 0, 3, 9, 3, 5, 5, 3, 7, -1, -1, -1, -1, -1, -1, -1},
    {9, 8, 7, 5, 9, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {5, 8, 4, 5, 10, 8, 10, 11, 8, -1, -1, -1, -1, -1, -1, -1},
    {5, 0, 4, 5, 11, 0, 5, 10, 11, 11, 3, 0, -1, -1, -1, -1},
    {0, 1, 9, 8, 4, 10, 8, 10, 11, 10, 4, 5, -1, -1, -1, -1},
    {10, 11, 4, 10, 4, 5, 11, 3, 4, 9, 4, 1, 3, 1, 4, -1},
    {2, 5, 1, 2, 8, 5, 2, 11, 8, 4, 5, 8, -1, -1, -1, -1},
    {0, 4, 11, 0, 11, 3, 4, 5, 11, 2, 11, 1, 5, 1, 11, -1},
    {0, 2, 5, 0, 5, 9, 2, 11, 5, 4, 5, 8, 11, 8, 5, -1},
    {9, 4, 5, 2, 11, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 5, 10, 3, 5, 2, 3, 4, 5, 3, 8, 4, -1, -1, -1, -1},
    {5, 10, 2, 5, 2, 4, 4, 2, 0, -1, -1, -1, -1, -1, -1, -1},
    {3, 10, 2, 3, 5, 10, 3, 8, 5, 4, 5, 8, 0, 1, 9, -1},
    {5, 10, 2, 5, 2, 4, 1, 9, 2, 9, 4, 2, -1, -1, -1, -1},
    {8, 4, 5, 8, 5, 3, 3, 5, 1, -1, -1, -1, -1, -1, -1, -1},
    {0, 4, 5, 1, 0, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 4, 5, 8, 5, 3, 9, 0, 5, 0, 3, 5, -1, -1, -1, -1},
    {9, 4, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 11, 7, 4, 9, 11, 9, 10, 11, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 4, 9, 7, 9, 11, 7, 9, 10, 11, -1, -1, -1, -1},
    {1, 10, 11, 1, 11, 4, 1, 4, 0, 7, 4, 11, -1, -1, -1, -1},
    {3, 1, 4, 3, 4, 8, 1, 10, 4, 7, 4, 11, 10, 11, 4, -1},
    {4, 11, 7, 9, 11, 4, 9, 2, 11, 9, 1, 2, -1, -1, -1, -1},
    {9, 7, 4, 9, 11, 7, 9, 1, 11, 2, 11, 1, 0, 8, 3, -1},
    {11, 7, 4, 11, 4, 2, 2, 4, 0, -1, -1, -1, -1, -1, -1, -1},
    {11, 7, 4, 11, 4, 2, 8, 3, 4, 3, 2, 4, -1, -1, -1, -1},
    {2, 9, 10, 2, 7, 9, 2, 3, 7, 7, 4, 9, -1, -1, -1, -1},
    {9, 10, 7, 9, 7, 4, 10, 2, 7, 8, 7, 0, 2, 0, 7, -1},
    {3, 7, 10, 3, 10, 2, 7, 4, 10, 1, 10, 0, 4, 0, 10, -1},
    {1, 10, 2, 8, 7, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 9, 1, 4, 1, 7, 7, 1, 3, -1, -1, -1, -1, -1, -1, -1},
    {4, 9, 1, 4, 1, 7, 0, 8, 1, 8, 7, 1, -1, -1, -1, -1},
    {4, 0, 3, 7, 4, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 8, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 10, 8, 10, 11, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 9, 3, 9, 11, 11, 9, 10, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 10, 0, 10, 8, 8, 10, 11, -1, -1, -1, -1, -1, -1, -1},
    {3, 1, 10, 11, 3, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 11, 1, 11, 9, 9, 11, 8, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 9, 3, 9, 11, 1, 2, 9, 2, 11, 9, -1, -1, -1, -1},
    {0, 2, 11, 8, 0, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 2, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 10, 10, 8, 9, -1, -1, -1, -1, -1, -1, -1},
    {9, 10, 2, 0, 9, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 10, 0, 1, 8, 1, 10, 8, -1, -1, -1, -1},
    {1, 10, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 3, 8, 9, 1, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1}};

// workspace: [0, 256) ticket; then the block status words; then per grid point: vertex offset, face offset (int32) and code (uint16:
// cube index in bits 0-7 (0 for points that start no cell), owned crossing axes in bits 8-10)
struct McWs {
    uint32_t* ticket;
    unsigned long long* status;
    int* voff;
    int* foff;
    uint16_t* code;
};

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

__host__ __device__ inline McWs mc_carve(void* ws, uint64_t npts) {
    const uint64_t nblk = (npts + kMcThreads - 1) / kMcThreads;
    char* p = (char*)ws;
    McWs w;
    w.ticket = (uint32_t*)p; p += 256;
    w.status = (unsigned long long*)p; p += align256(nblk * 8);
    w.voff = (int*)p; p += align256(npts * 4);
    w.foff = (int*)p; p += align256(npts * 4);
    w.code = (uint16_t*)p;
    return w;
}

// status word of a block: bits 62-63 state (1 = block aggregate, 2 = inclusive prefix), bits 31-61 faces, bits 0-30 vertices.
// The host bounds 3 * points and 5 * cells by INT32_MAX, so both totals fit their 31-bit fields.
constexpr unsigned long long kAgg = 1ull << 62, kPrefix = 2ull << 62, kVal = (1ull << 62) - 1;
__device__ __forceinline__ unsigned long long pack_vf(uint32_t v, uint32_t f) { return (unsigned long long)v | ((unsigned long long)f << 31); }

__device__ __forceinline__ float eff_iso(float iso, const float* iso_dev) { return iso_dev ? fminf(iso, *iso_dev) : iso; }

__global__ void __launch_bounds__(kMcThreads)
k_mc_count(const float* __restrict__ vol, uint32_t nx, uint32_t ny, uint32_t nz, float iso, const float* __restrict__ iso_dev, McWs w,
           int* __restrict__ counts) {
    __shared__ uint32_t s_bid;
    __shared__ unsigned long long s_warp[kMcThreads / 32], s_prefix;
    if (threadIdx.x == 0) s_bid = atomicAdd(w.ticket, 1u);            // blocks start in ticket order: every predecessor is running
    __syncthreads();
    const uint32_t bid = s_bid, nblk = gridDim.x;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t npts = (uint64_t)nx * ny * nz;
    const uint64_t p = (uint64_t)bid * kMcThreads + threadIdx.x;
    const float th = eff_iso(iso, iso_dev);
    uint32_t nv = 0, nf = 0, code = 0;
    if (p < npts) {
        const uint64_t syz = (uint64_t)ny * nz;
        const uint32_t i = (uint32_t)(p / syz), j = (uint32_t)((p / nz) % ny), k = (uint32_t)(p % nz);
        const bool in = vol[p] > th;
        const bool cx = i + 1 < nx, cy = j + 1 < ny, cz = k + 1 < nz;
        if (cx && (vol[p + syz] > th) != in) code |= 1u << 8;
        if (cy && (vol[p + nz] > th) != in) code |= 2u << 8;
        if (cz && (vol[p + 1] > th) != in) code |= 4u << 8;
        nv = __popc(code);
        if (cx && cy && cz) {
            uint32_t ci = 0;
            #pragma unroll
            for (int m = 0; m < 8; m++) {
                const uint64_t q = p + c_corner[m][0] * syz + c_corner[m][1] * nz + c_corner[m][2];
                if (!(vol[q] > th)) ci |= 1u << m;
            }
            code |= ci;
            for (int t = 0; t < 15 && c_tri[ci][t] >= 0; t += 3) nf++;
        }
    }
    // block exclusive scan of (nv, nf), packed in one 64-bit word (per-block sums stay far below 2^31)
    const unsigned long long mine = pack_vf(nv, nf);
    unsigned long long incl = mine;
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) { unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (uint32_t)o) incl += v; }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    unsigned long long warp_base = 0, block_tot = 0;
    #pragma unroll
    for (int q = 0; q < kMcThreads / 32; q++) { if (q < (int)wid) warp_base += s_warp[q]; block_tot += s_warp[q]; }
    volatile unsigned long long* status = w.status;
    if (wid == 0) {
        unsigned long long excl = 0;
        if (bid == 0) {
            if (lane == 0) status[0] = kPrefix | block_tot;
        } else {
            if (lane == 0) status[bid] = kAgg | block_tot;
            // decoupled look-back: scan the predecessors 32 at a time, nearest first, until one has published its inclusive prefix
            int64_t base = (int64_t)bid - 1;
            while (true) {
                const int64_t j = base - (int64_t)lane;
                unsigned long long s = kPrefix;                         // before block 0: an inclusive prefix of zero
                if (j >= 0) { do { s = status[j]; } while ((s >> 62) == 0); }
                const uint32_t pm = __ballot_sync(0xffffffffu, (s >> 62) == 2);
                const uint32_t stop = pm ? (uint32_t)(__ffs(pm) - 1) : 31u;
                unsigned long long v = lane <= stop ? (s & kVal) : 0ull;
                #pragma unroll
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                excl += v;
                if (pm) break;
                base -= 32;
            }
            if (lane == 0) status[bid] = kPrefix | (excl + block_tot);
        }
        if (lane == 0) s_prefix = excl;
    }
    __syncthreads();
    const unsigned long long off = s_prefix + warp_base + incl - mine;
    if (p < npts) {
        w.voff[p] = (int)(off & 0x7fffffffull);
        w.foff[p] = (int)((off >> 31) & 0x7fffffffull);
        w.code[p] = (uint16_t)code;
    }
    if (bid == nblk - 1 && threadIdx.x == 0) {
        const unsigned long long tot = s_prefix + block_tot;
        counts[0] = (int)(tot & 0x7fffffffull);
        counts[1] = (int)((tot >> 31) & 0x7fffffffull);
    }
}

__global__ void __launch_bounds__(kMcThreads)
k_mc_emit(const float* __restrict__ vol, uint32_t nx, uint32_t ny, uint32_t nz, float iso, const float* __restrict__ iso_dev, McWs w,
          float scale, float offset, float* __restrict__ vertices, int* __restrict__ faces) {
    const uint64_t npts = (uint64_t)nx * ny * nz;
    const uint64_t p = (uint64_t)blockIdx.x * kMcThreads + threadIdx.x;
    if (p >= npts) return;
    const uint32_t code = w.code[p];
    const uint32_t emask = code >> 8, ci = code & 0xffu;
    if (emask == 0 && ci == 0) return;
    const uint64_t syz = (uint64_t)ny * nz;
    const uint32_t i = (uint32_t)(p / syz), j = (uint32_t)((p / nz) % ny), k = (uint32_t)(p % nz);
    if (emask) {
        const float th = eff_iso(iso, iso_dev);
        const float s = vol[p];
        const uint64_t stride[3] = {syz, nz, 1};
        const float base[3] = {(float)i, (float)j, (float)k};
        int vid = w.voff[p];
        #pragma unroll
        for (int a = 0; a < 3; a++) {
            if (!(emask & (1u << a))) continue;
            const float t = (th - s) / (vol[p + stride[a]] - s);
            float v[3] = {base[0], base[1], base[2]};
            v[a] = v[a] + t;
            float* o = vertices + 3 * (size_t)vid;
            o[0] = v[0] * scale + offset; o[1] = v[1] * scale + offset; o[2] = v[2] * scale + offset;
            vid++;
        }
    }
    if (ci != 0) {
        int* o = faces + 3 * (size_t)w.foff[p];
        for (int t = 0; t < 15 && c_tri[ci][t] >= 0; t++) {
            const int e = c_tri[ci][t];
            const int m = c_edge_from[e], a = c_edge_axis[e];
            const uint64_t q = p + c_corner[m][0] * syz + c_corner[m][1] * nz + c_corner[m][2];
            o[t] = w.voff[q] + __popc((w.code[q] >> 8) & ((1u << a) - 1u));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Texture atlas texels (layout: nerf/mesh.py::atlas_layout, oracle/mesh_ref.py).  Faces 2p and 2p+1 share the c x c cell p at
// (p % n, p / n); UV corners, in texel units from the cell origin: face 2p (1,1), (c-3,1), (1,c-3); face 2p+1 (c-1,c-1), (3,c-1),
// (c-1,3).  A texel belongs to a face iff its centre is at Chebyshev distance < 1 from the face's UV triangle; with texel centres at
// half-integers (i + 0.5, j + 0.5) in the cell that is  i, j <= c-3, i+j <= c-2  (even face)  or  i, j >= 2, i+j >= c  (odd face).
// ---------------------------------------------------------------------------------------------------------------------------
__global__ void k_atlas_texels(const float* __restrict__ vertices, const int* __restrict__ faces, uint32_t F, uint32_t T, uint32_t c,
                               uint32_t n, float bound, float* __restrict__ points, int* __restrict__ owner, float* __restrict__ vt) {
    const uint64_t idx = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (uint64_t)T * T) return;
    // the 3F texture coordinates (3F < T^2 because T >= 8n and F <= 2n^2)
    if (idx < 3ull * F) {
        const uint32_t f = (uint32_t)(idx / 3), corner = (uint32_t)(idx % 3), cell = f >> 1;
        // even face: (1,1), (c-3,1), (1,c-3); odd face: (c-1,c-1), (3,c-1), (c-1,3)
        const uint32_t lu = (f & 1) ? (corner == 1 ? 3u : c - 1) : (corner == 1 ? c - 3 : 1u);
        const uint32_t lv = (f & 1) ? (corner == 2 ? 3u : c - 1) : (corner == 2 ? c - 3 : 1u);
        vt[2 * idx] = ((float)((cell % n) * c) + (float)lu) / (float)T;
        vt[2 * idx + 1] = ((float)((cell / n) * c) + (float)lv) / (float)T;
    }
    const uint32_t r = (uint32_t)(idx / T), x = (uint32_t)(idx % T);
    const uint32_t px = x / c, py = r / c;
    int f = -1;
    const uint32_t i = x - px * c, j = r - py * c, cell = py * n + px;
    if (px < n && py < n) {
        if (i + 3 <= c && j + 3 <= c && i + j + 2 <= c) { if (2ull * cell < F) f = (int)(2 * cell); }
        else if (i >= 2 && j >= 2 && i + j >= c) { if (2ull * cell + 1 < F) f = (int)(2 * cell + 1); }
    }
    float3 out = make_float3(0.f, 0.f, 0.f);
    if (f >= 0) {
        const float li = (float)i + 0.5f, lj = (float)j + 0.5f, d = (float)(c - 4);
        float b1, b2;
        if (f & 1) { b1 = ((float)(c - 1) - li) / d; b2 = ((float)(c - 1) - lj) / d; }
        else { b1 = (li - 1.f) / d; b2 = (lj - 1.f) / d; }
        const int* fv = faces + 3 * (size_t)f;
        const float* v0 = vertices + 3 * (size_t)fv[0];
        const float* v1 = vertices + 3 * (size_t)fv[1];
        const float* v2 = vertices + 3 * (size_t)fv[2];
        float q[3];
        #pragma unroll
        for (int a = 0; a < 3; a++) q[a] = mi3d_clampf((v0[a] + b1 * (v1[a] - v0[a])) + b2 * (v2[a] - v0[a]), -bound, bound);
        out = make_float3(q[0], q[1], q[2]);
    }
    points[3 * idx] = out.x; points[3 * idx + 1] = out.y; points[3 * idx + 2] = out.z;
    owner[idx] = f;
}

bool mc_dims_ok(uint32_t nx, uint32_t ny, uint32_t nz) {
    if (nx < 2 || ny < 2 || nz < 2) return false;
    const uint64_t npts = (uint64_t)nx * ny * nz, ncells = (uint64_t)(nx - 1) * (ny - 1) * (nz - 1);
    return 3 * npts <= 0x7fffffffull && 5 * ncells <= 0x7fffffffull;      // every vertex / face index fits int32
}

}  // namespace

extern "C" {

size_t mi3d_mc_workspace_bytes(uint32_t nx, uint32_t ny, uint32_t nz) {
    if (!mc_dims_ok(nx, ny, nz)) return 0;
    const uint64_t npts = (uint64_t)nx * ny * nz, nblk = (npts + kMcThreads - 1) / kMcThreads;
    return 256 + align256(nblk * 8) + 2 * align256(npts * 4) + align256(npts * 2);
}

int mi3d_mc_count(const float* volume, uint32_t nx, uint32_t ny, uint32_t nz, float iso, const float* iso_dev, void* workspace,
                  int* counts, mi3d_stream_t stream) {
    if (!volume || !workspace || !counts || !mc_dims_ok(nx, ny, nz)) return MI3D_ERR_ARG;
    const uint64_t npts = (uint64_t)nx * ny * nz, nblk = (npts + kMcThreads - 1) / kMcThreads;
    cudaStream_t st = (cudaStream_t)stream;
    MI3D_CHECK(cudaMemsetAsync(workspace, 0, 256 + align256(nblk * 8), st));        // ticket + status words
    k_mc_count<<<(unsigned)nblk, kMcThreads, 0, st>>>(volume, nx, ny, nz, iso, iso_dev, mc_carve(workspace, npts), counts);
    MI3D_RETURN_LAUNCH();
}

int mi3d_mc_emit(const float* volume, uint32_t nx, uint32_t ny, uint32_t nz, float iso, const float* iso_dev, const void* workspace,
                 float scale, float offset, float* vertices, int* faces, mi3d_stream_t stream) {
    if (!volume || !workspace || !vertices || !faces || !mc_dims_ok(nx, ny, nz)) return MI3D_ERR_ARG;
    const uint64_t npts = (uint64_t)nx * ny * nz, nblk = (npts + kMcThreads - 1) / kMcThreads;
    k_mc_emit<<<(unsigned)nblk, kMcThreads, 0, (cudaStream_t)stream>>>(volume, nx, ny, nz, iso, iso_dev, mc_carve((void*)workspace, npts),
                                                                        scale, offset, vertices, faces);
    MI3D_RETURN_LAUNCH();
}

int mi3d_mesh_atlas_texels(const float* vertices, const int* faces, uint32_t F, uint32_t T, uint32_t c, uint32_t n, float bound,
                           float* points, int* owner, float* vt, mi3d_stream_t stream) {
    if (!vertices || !faces || !points || !owner || !vt || F == 0 || c < 8 || n == 0 || (uint64_t)n * c > T) return MI3D_ERR_ARG;
    if ((uint64_t)n * n * 2 < F || (uint64_t)F > 0x7fffffffull) return MI3D_ERR_ARG;
    const uint64_t total = (uint64_t)T * T;
    k_atlas_texels<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(vertices, faces, F, T, c, n, bound, points, owner, vt);
    MI3D_RETURN_LAUNCH();
}

}  // extern "C"
