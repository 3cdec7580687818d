"""numpy restatement of the native mesh export (csrc/mesh.cu, nerf/mesh.py): marching cubes and the per-face texture atlas.

Marching cubes is the Lorensen-Cline algorithm with the public-domain 256-case triangle table of Paul Bourke / Cory Bloyd (the
table PyMCubes uses), carried here as an independent copy of the one in csrc/mesh.cu.  The contract both follow:
  * volume fp32 [nx, ny, nz], C order, index (i, j, k) <-> (x, y, z); a corner is inside iff sigma > iso (iso rounded to fp32)
  * cube index bit m set iff corner m (Bourke numbering) is NOT inside
  * one vertex per crossing grid edge, owned by its lower end point p, at p + t e_a with t = (iso - s_p) / (s_{p+e_a} - s_p) in
    fp32 (single roundings, no FMA); numbering: grid points in C order, then axis x < y < z within a point
  * faces: cells in C order, triangles in table order; the table's winding puts the right-hand normal on the side of the corners
    with sigma <= iso, i.e. out of the solid, so triangles are emitted as written
  * optional output affine map v * scale + offset (fp32, two roundings)
"""
import math

import numpy as np

# corner m -> (dx, dy, dz)
CORNERS = np.array([(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)], np.int64)
# edge e -> (corner a, corner b); the edge runs from a along +axis to b
EDGE_CORNERS = np.array([(0, 1), (1, 2), (3, 2), (0, 3), (4, 5), (5, 6), (7, 6), (4, 7), (0, 4), (1, 5), (2, 6), (3, 7)], np.int64)
EDGE_AXIS = np.array([0, 1, 0, 1, 0, 1, 0, 1, 2, 2, 2, 2], np.int64)

TRI_TABLE = [
    [],
    [0, 8, 3],
    [0, 1, 9],
    [1, 8, 3, 9, 8, 1],
    [1, 2, 10],
    [0, 8, 3, 1, 2, 10],
    [9, 2, 10, 0, 2, 9],
    [2, 8, 3, 2, 10, 8, 10, 9, 8],
    [3, 11, 2],
    [0, 11, 2, 8, 11, 0],
    [1, 9, 0, 2, 3, 11],
    [1, 11, 2, 1, 9, 11, 9, 8, 11],
    [3, 10, 1, 11, 10, 3],
    [0, 10, 1, 0, 8, 10, 8, 11, 10],
    [3, 9, 0, 3, 11, 9, 11, 10, 9],
    [9, 8, 10, 10, 8, 11],
    [4, 7, 8],
    [4, 3, 0, 7, 3, 4],
    [0, 1, 9, 8, 4, 7],
    [4, 1, 9, 4, 7, 1, 7, 3, 1],
    [1, 2, 10, 8, 4, 7],
    [3, 4, 7, 3, 0, 4, 1, 2, 10],
    [9, 2, 10, 9, 0, 2, 8, 4, 7],
    [2, 10, 9, 2, 9, 7, 2, 7, 3, 7, 9, 4],
    [8, 4, 7, 3, 11, 2],
    [11, 4, 7, 11, 2, 4, 2, 0, 4],
    [9, 0, 1, 8, 4, 7, 2, 3, 11],
    [4, 7, 11, 9, 4, 11, 9, 11, 2, 9, 2, 1],
    [3, 10, 1, 3, 11, 10, 7, 8, 4],
    [1, 11, 10, 1, 4, 11, 1, 0, 4, 7, 11, 4],
    [4, 7, 8, 9, 0, 11, 9, 11, 10, 11, 0, 3],
    [4, 7, 11, 4, 11, 9, 9, 11, 10],
    [9, 5, 4],
    [9, 5, 4, 0, 8, 3],
    [0, 5, 4, 1, 5, 0],
    [8, 5, 4, 8, 3, 5, 3, 1, 5],
    [1, 2, 10, 9, 5, 4],
    [3, 0, 8, 1, 2, 10, 4, 9, 5],
    [5, 2, 10, 5, 4, 2, 4, 0, 2],
    [2, 10, 5, 3, 2, 5, 3, 5, 4, 3, 4, 8],
    [9, 5, 4, 2, 3, 11],
    [0, 11, 2, 0, 8, 11, 4, 9, 5],
    [0, 5, 4, 0, 1, 5, 2, 3, 11],
    [2, 1, 5, 2, 5, 8, 2, 8, 11, 4, 8, 5],
    [10, 3, 11, 10, 1, 3, 9, 5, 4],
    [4, 9, 5, 0, 8, 1, 8, 10, 1, 8, 11, 10],
    [5, 4, 0, 5, 0, 11, 5, 11, 10, 11, 0, 3],
    [5, 4, 8, 5, 8, 10, 10, 8, 11],
    [9, 7, 8, 5, 7, 9],
    [9, 3, 0, 9, 5, 3, 5, 7, 3],
    [0, 7, 8, 0, 1, 7, 1, 5, 7],
    [1, 5, 3, 3, 5, 7],
    [9, 7, 8, 9, 5, 7, 10, 1, 2],
    [10, 1, 2, 9, 5, 0, 5, 3, 0, 5, 7, 3],
    [8, 0, 2, 8, 2, 5, 8, 5, 7, 10, 5, 2],
    [2, 10, 5, 2, 5, 3, 3, 5, 7],
    [7, 9, 5, 7, 8, 9, 3, 11, 2],
    [9, 5, 7, 9, 7, 2, 9, 2, 0, 2, 7, 11],
    [2, 3, 11, 0, 1, 8, 1, 7, 8, 1, 5, 7],
    [11, 2, 1, 11, 1, 7, 7, 1, 5],
    [9, 5, 8, 8, 5, 7, 10, 1, 3, 10, 3, 11],
    [5, 7, 0, 5, 0, 9, 7, 11, 0, 1, 0, 10, 11, 10, 0],
    [11, 10, 0, 11, 0, 3, 10, 5, 0, 8, 0, 7, 5, 7, 0],
    [11, 10, 5, 7, 11, 5],
    [10, 6, 5],
    [0, 8, 3, 5, 10, 6],
    [9, 0, 1, 5, 10, 6],
    [1, 8, 3, 1, 9, 8, 5, 10, 6],
    [1, 6, 5, 2, 6, 1],
    [1, 6, 5, 1, 2, 6, 3, 0, 8],
    [9, 6, 5, 9, 0, 6, 0, 2, 6],
    [5, 9, 8, 5, 8, 2, 5, 2, 6, 3, 2, 8],
    [2, 3, 11, 10, 6, 5],
    [11, 0, 8, 11, 2, 0, 10, 6, 5],
    [0, 1, 9, 2, 3, 11, 5, 10, 6],
    [5, 10, 6, 1, 9, 2, 9, 11, 2, 9, 8, 11],
    [6, 3, 11, 6, 5, 3, 5, 1, 3],
    [0, 8, 11, 0, 11, 5, 0, 5, 1, 5, 11, 6],
    [3, 11, 6, 0, 3, 6, 0, 6, 5, 0, 5, 9],
    [6, 5, 9, 6, 9, 11, 11, 9, 8],
    [5, 10, 6, 4, 7, 8],
    [4, 3, 0, 4, 7, 3, 6, 5, 10],
    [1, 9, 0, 5, 10, 6, 8, 4, 7],
    [10, 6, 5, 1, 9, 7, 1, 7, 3, 7, 9, 4],
    [6, 1, 2, 6, 5, 1, 4, 7, 8],
    [1, 2, 5, 5, 2, 6, 3, 0, 4, 3, 4, 7],
    [8, 4, 7, 9, 0, 5, 0, 6, 5, 0, 2, 6],
    [7, 3, 9, 7, 9, 4, 3, 2, 9, 5, 9, 6, 2, 6, 9],
    [3, 11, 2, 7, 8, 4, 10, 6, 5],
    [5, 10, 6, 4, 7, 2, 4, 2, 0, 2, 7, 11],
    [0, 1, 9, 4, 7, 8, 2, 3, 11, 5, 10, 6],
    [9, 2, 1, 9, 11, 2, 9, 4, 11, 7, 11, 4, 5, 10, 6],
    [8, 4, 7, 3, 11, 5, 3, 5, 1, 5, 11, 6],
    [5, 1, 11, 5, 11, 6, 1, 0, 11, 7, 11, 4, 0, 4, 11],
    [0, 5, 9, 0, 6, 5, 0, 3, 6, 11, 6, 3, 8, 4, 7],
    [6, 5, 9, 6, 9, 11, 4, 7, 9, 7, 11, 9],
    [10, 4, 9, 6, 4, 10],
    [4, 10, 6, 4, 9, 10, 0, 8, 3],
    [10, 0, 1, 10, 6, 0, 6, 4, 0],
    [8, 3, 1, 8, 1, 6, 8, 6, 4, 6, 1, 10],
    [1, 4, 9, 1, 2, 4, 2, 6, 4],
    [3, 0, 8, 1, 2, 9, 2, 4, 9, 2, 6, 4],
    [0, 2, 4, 4, 2, 6],
    [8, 3, 2, 8, 2, 4, 4, 2, 6],
    [10, 4, 9, 10, 6, 4, 11, 2, 3],
    [0, 8, 2, 2, 8, 11, 4, 9, 10, 4, 10, 6],
    [3, 11, 2, 0, 1, 6, 0, 6, 4, 6, 1, 10],
    [6, 4, 1, 6, 1, 10, 4, 8, 1, 2, 1, 11, 8, 11, 1],
    [9, 6, 4, 9, 3, 6, 9, 1, 3, 11, 6, 3],
    [8, 11, 1, 8, 1, 0, 11, 6, 1, 9, 1, 4, 6, 4, 1],
    [3, 11, 6, 3, 6, 0, 0, 6, 4],
    [6, 4, 8, 11, 6, 8],
    [7, 10, 6, 7, 8, 10, 8, 9, 10],
    [0, 7, 3, 0, 10, 7, 0, 9, 10, 6, 7, 10],
    [10, 6, 7, 1, 10, 7, 1, 7, 8, 1, 8, 0],
    [10, 6, 7, 10, 7, 1, 1, 7, 3],
    [1, 2, 6, 1, 6, 8, 1, 8, 9, 8, 6, 7],
    [2, 6, 9, 2, 9, 1, 6, 7, 9, 0, 9, 3, 7, 3, 9],
    [7, 8, 0, 7, 0, 6, 6, 0, 2],
    [7, 3, 2, 6, 7, 2],
    [2, 3, 11, 10, 6, 8, 10, 8, 9, 8, 6, 7],
    [2, 0, 7, 2, 7, 11, 0, 9, 7, 6, 7, 10, 9, 10, 7],
    [1, 8, 0, 1, 7, 8, 1, 10, 7, 6, 7, 10, 2, 3, 11],
    [11, 2, 1, 11, 1, 7, 10, 6, 1, 6, 7, 1],
    [8, 9, 6, 8, 6, 7, 9, 1, 6, 11, 6, 3, 1, 3, 6],
    [0, 9, 1, 11, 6, 7],
    [7, 8, 0, 7, 0, 6, 3, 11, 0, 11, 6, 0],
    [7, 11, 6],
    [7, 6, 11],
    [3, 0, 8, 11, 7, 6],
    [0, 1, 9, 11, 7, 6],
    [8, 1, 9, 8, 3, 1, 11, 7, 6],
    [10, 1, 2, 6, 11, 7],
    [1, 2, 10, 3, 0, 8, 6, 11, 7],
    [2, 9, 0, 2, 10, 9, 6, 11, 7],
    [6, 11, 7, 2, 10, 3, 10, 8, 3, 10, 9, 8],
    [7, 2, 3, 6, 2, 7],
    [7, 0, 8, 7, 6, 0, 6, 2, 0],
    [2, 7, 6, 2, 3, 7, 0, 1, 9],
    [1, 6, 2, 1, 8, 6, 1, 9, 8, 8, 7, 6],
    [10, 7, 6, 10, 1, 7, 1, 3, 7],
    [10, 7, 6, 1, 7, 10, 1, 8, 7, 1, 0, 8],
    [0, 3, 7, 0, 7, 10, 0, 10, 9, 6, 10, 7],
    [7, 6, 10, 7, 10, 8, 8, 10, 9],
    [6, 8, 4, 11, 8, 6],
    [3, 6, 11, 3, 0, 6, 0, 4, 6],
    [8, 6, 11, 8, 4, 6, 9, 0, 1],
    [9, 4, 6, 9, 6, 3, 9, 3, 1, 11, 3, 6],
    [6, 8, 4, 6, 11, 8, 2, 10, 1],
    [1, 2, 10, 3, 0, 11, 0, 6, 11, 0, 4, 6],
    [4, 11, 8, 4, 6, 11, 0, 2, 9, 2, 10, 9],
    [10, 9, 3, 10, 3, 2, 9, 4, 3, 11, 3, 6, 4, 6, 3],
    [8, 2, 3, 8, 4, 2, 4, 6, 2],
    [0, 4, 2, 4, 6, 2],
    [1, 9, 0, 2, 3, 4, 2, 4, 6, 4, 3, 8],
    [1, 9, 4, 1, 4, 2, 2, 4, 6],
    [8, 1, 3, 8, 6, 1, 8, 4, 6, 6, 10, 1],
    [10, 1, 0, 10, 0, 6, 6, 0, 4],
    [4, 6, 3, 4, 3, 8, 6, 10, 3, 0, 3, 9, 10, 9, 3],
    [10, 9, 4, 6, 10, 4],
    [4, 9, 5, 7, 6, 11],
    [0, 8, 3, 4, 9, 5, 11, 7, 6],
    [5, 0, 1, 5, 4, 0, 7, 6, 11],
    [11, 7, 6, 8, 3, 4, 3, 5, 4, 3, 1, 5],
    [9, 5, 4, 10, 1, 2, 7, 6, 11],
    [6, 11, 7, 1, 2, 10, 0, 8, 3, 4, 9, 5],
    [7, 6, 11, 5, 4, 10, 4, 2, 10, 4, 0, 2],
    [3, 4, 8, 3, 5, 4, 3, 2, 5, 10, 5, 2, 11, 7, 6],
    [7, 2, 3, 7, 6, 2, 5, 4, 9],
    [9, 5, 4, 0, 8, 6, 0, 6, 2, 6, 8, 7],
    [3, 6, 2, 3, 7, 6, 1, 5, 0, 5, 4, 0],
    [6, 2, 8, 6, 8, 7, 2, 1, 8, 4, 8, 5, 1, 5, 8],
    [9, 5, 4, 10, 1, 6, 1, 7, 6, 1, 3, 7],
    [1, 6, 10, 1, 7, 6, 1, 0, 7, 8, 7, 0, 9, 5, 4],
    [4, 0, 10, 4, 10, 5, 0, 3, 10, 6, 10, 7, 3, 7, 10],
    [7, 6, 10, 7, 10, 8, 5, 4, 10, 4, 8, 10],
    [6, 9, 5, 6, 11, 9, 11, 8, 9],
    [3, 6, 11, 0, 6, 3, 0, 5, 6, 0, 9, 5],
    [0, 11, 8, 0, 5, 11, 0, 1, 5, 5, 6, 11],
    [6, 11, 3, 6, 3, 5, 5, 3, 1],
    [1, 2, 10, 9, 5, 11, 9, 11, 8, 11, 5, 6],
    [0, 11, 3, 0, 6, 11, 0, 9, 6, 5, 6, 9, 1, 2, 10],
    [11, 8, 5, 11, 5, 6, 8, 0, 5, 10, 5, 2, 0, 2, 5],
    [6, 11, 3, 6, 3, 5, 2, 10, 3, 10, 5, 3],
    [5, 8, 9, 5, 2, 8, 5, 6, 2, 3, 8, 2],
    [9, 5, 6, 9, 6, 0, 0, 6, 2],
    [1, 5, 8, 1, 8, 0, 5, 6, 8, 3, 8, 2, 6, 2, 8],
    [1, 5, 6, 2, 1, 6],
    [1, 3, 6, 1, 6, 10, 3, 8, 6, 5, 6, 9, 8, 9, 6],
    [10, 1, 0, 10, 0, 6, 9, 5, 0, 5, 6, 0],
    [0, 3, 8, 5, 6, 10],
    [10, 5, 6],
    [11, 5, 10, 7, 5, 11],
    [11, 5, 10, 11, 7, 5, 8, 3, 0],
    [5, 11, 7, 5, 10, 11, 1, 9, 0],
    [10, 7, 5, 10, 11, 7, 9, 8, 1, 8, 3, 1],
    [11, 1, 2, 11, 7, 1, 7, 5, 1],
    [0, 8, 3, 1, 2, 7, 1, 7, 5, 7, 2, 11],
    [9, 7, 5, 9, 2, 7, 9, 0, 2, 2, 11, 7],
    [7, 5, 2, 7, 2, 11, 5, 9, 2, 3, 2, 8, 9, 8, 2],
    [2, 5, 10, 2, 3, 5, 3, 7, 5],
    [8, 2, 0, 8, 5, 2, 8, 7, 5, 10, 2, 5],
    [9, 0, 1, 5, 10, 3, 5, 3, 7, 3, 10, 2],
    [9, 8, 2, 9, 2, 1, 8, 7, 2, 10, 2, 5, 7, 5, 2],
    [1, 3, 5, 3, 7, 5],
    [0, 8, 7, 0, 7, 1, 1, 7, 5],
    [9, 0, 3, 9, 3, 5, 5, 3, 7],
    [9, 8, 7, 5, 9, 7],
    [5, 8, 4, 5, 10, 8, 10, 11, 8],
    [5, 0, 4, 5, 11, 0, 5, 10, 11, 11, 3, 0],
    [0, 1, 9, 8, 4, 10, 8, 10, 11, 10, 4, 5],
    [10, 11, 4, 10, 4, 5, 11, 3, 4, 9, 4, 1, 3, 1, 4],
    [2, 5, 1, 2, 8, 5, 2, 11, 8, 4, 5, 8],
    [0, 4, 11, 0, 11, 3, 4, 5, 11, 2, 11, 1, 5, 1, 11],
    [0, 2, 5, 0, 5, 9, 2, 11, 5, 4, 5, 8, 11, 8, 5],
    [9, 4, 5, 2, 11, 3],
    [2, 5, 10, 3, 5, 2, 3, 4, 5, 3, 8, 4],
    [5, 10, 2, 5, 2, 4, 4, 2, 0],
    [3, 10, 2, 3, 5, 10, 3, 8, 5, 4, 5, 8, 0, 1, 9],
    [5, 10, 2, 5, 2, 4, 1, 9, 2, 9, 4, 2],
    [8, 4, 5, 8, 5, 3, 3, 5, 1],
    [0, 4, 5, 1, 0, 5],
    [8, 4, 5, 8, 5, 3, 9, 0, 5, 0, 3, 5],
    [9, 4, 5],
    [4, 11, 7, 4, 9, 11, 9, 10, 11],
    [0, 8, 3, 4, 9, 7, 9, 11, 7, 9, 10, 11],
    [1, 10, 11, 1, 11, 4, 1, 4, 0, 7, 4, 11],
    [3, 1, 4, 3, 4, 8, 1, 10, 4, 7, 4, 11, 10, 11, 4],
    [4, 11, 7, 9, 11, 4, 9, 2, 11, 9, 1, 2],
    [9, 7, 4, 9, 11, 7, 9, 1, 11, 2, 11, 1, 0, 8, 3],
    [11, 7, 4, 11, 4, 2, 2, 4, 0],
    [11, 7, 4, 11, 4, 2, 8, 3, 4, 3, 2, 4],
    [2, 9, 10, 2, 7, 9, 2, 3, 7, 7, 4, 9],
    [9, 10, 7, 9, 7, 4, 10, 2, 7, 8, 7, 0, 2, 0, 7],
    [3, 7, 10, 3, 10, 2, 7, 4, 10, 1, 10, 0, 4, 0, 10],
    [1, 10, 2, 8, 7, 4],
    [4, 9, 1, 4, 1, 7, 7, 1, 3],
    [4, 9, 1, 4, 1, 7, 0, 8, 1, 8, 7, 1],
    [4, 0, 3, 7, 4, 3],
    [4, 8, 7],
    [9, 10, 8, 10, 11, 8],
    [3, 0, 9, 3, 9, 11, 11, 9, 10],
    [0, 1, 10, 0, 10, 8, 8, 10, 11],
    [3, 1, 10, 11, 3, 10],
    [1, 2, 11, 1, 11, 9, 9, 11, 8],
    [3, 0, 9, 3, 9, 11, 1, 2, 9, 2, 11, 9],
    [0, 2, 11, 8, 0, 11],
    [3, 2, 11],
    [2, 3, 8, 2, 8, 10, 10, 8, 9],
    [9, 10, 2, 0, 9, 2],
    [2, 3, 8, 2, 8, 10, 0, 1, 8, 1, 10, 8],
    [1, 10, 2],
    [1, 3, 8, 9, 1, 8],
    [0, 9, 1],
    [0, 3, 8],
    [],
]
assert len(TRI_TABLE) == 256


def _tri_array():
    t = np.full((256, 5, 3), -1, np.int64)
    for ci, row in enumerate(TRI_TABLE):
        for k in range(len(row) // 3):
            t[ci, k] = row[3 * k:3 * k + 3]
    return t


_TRI = _tri_array()


def marching_cubes(vol, iso, scale=1.0, offset=0.0):
    """-> (vertices float32 [V,3], faces int32 [F,3]) under the contract of the module docstring."""
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    if vol.ndim != 3 or min(vol.shape) < 2:
        raise ValueError("volume must be 3-D with every dimension >= 2")
    nx, ny, nz = vol.shape
    iso = np.float32(iso)
    inside = vol > iso
    # crossing edges owned by each grid point, axis x < y < z
    cross = np.zeros((nx, ny, nz, 3), bool)
    cross[:-1, :, :, 0] = inside[:-1] != inside[1:]
    cross[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    cross[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = cross.reshape(-1)
    vid = np.cumsum(flat) - 1                                   # vertex id of each crossing (point-major, axis-minor)
    vid = vid.reshape(nx, ny, nz, 3)
    pi, ai = np.nonzero(flat.reshape(-1, 3))
    ijk = np.stack(np.unravel_index(pi, (nx, ny, nz)), axis=-1)
    s0 = vol.reshape(-1)[pi]
    nb = ijk.copy()
    nb[np.arange(len(ai)), ai] += 1
    s1 = vol[nb[:, 0], nb[:, 1], nb[:, 2]]
    t = (iso - s0) / (s1 - s0)                                  # fp32, one rounding per op
    verts = ijk.astype(np.float32)
    verts[np.arange(len(ai)), ai] = verts[np.arange(len(ai)), ai] + t
    scale, offset = np.float32(scale), np.float32(offset)
    if scale != 1 or offset != 0:
        verts = verts * scale + offset
    # faces
    ci = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for m, (dx, dy, dz) in enumerate(CORNERS):
        ci |= (~inside[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz]).astype(np.int64) << m
    cells = np.stack(np.nonzero((ci != 0) & (ci != 255)), axis=-1)            # C order
    tri = _TRI[ci[cells[:, 0], cells[:, 1], cells[:, 2]]]                     # [nc, 5, 3] edge ids
    keep = tri[:, :, 0] >= 0
    cell_of = np.broadcast_to(cells[:, None, None, :], tri.shape + (3,))[keep]   # [F, 3, 3]
    edges = tri[keep]                                                           # [F, 3]
    owner = cell_of + CORNERS[EDGE_CORNERS[edges, 0]]
    faces = vid[owner[..., 0], owner[..., 1], owner[..., 2], EDGE_AXIS[edges]]
    return verts.astype(np.float32), faces.astype(np.int32).reshape(-1, 3)


# ---------------------------------------------------------------------------------------------------------------------------
# Texture atlas: faces 2p and 2p+1 share square cell p of side c texels; cells fill rows of n.  UV corners in texel units relative
# to the cell origin: face 2p (1,1), (c-3,1), (1,c-3); face 2p+1 (c-1,c-1), (3,c-1), (c-1,3).  u runs along texel columns, v along
# rows; texel row r <-> v = (r + 0.5) / T.
# ---------------------------------------------------------------------------------------------------------------------------
ATLAS_T0, ATLAS_T_MAX, ATLAS_MIN_CELL = 2048, 16384, 8


def atlas_layout(F):
    """-> (T, c, n).  Raises ValueError past T = 16384."""
    if F < 1:
        raise ValueError("atlas needs at least one face")
    P = (F + 1) // 2
    n = math.isqrt(P)
    if n * n < P:
        n += 1
    T = ATLAS_T0
    while T // n < ATLAS_MIN_CELL:
        T *= 2
        if T > ATLAS_T_MAX:
            raise ValueError(f"{F} faces need a texture larger than {ATLAS_T_MAX}^2")
    return T, T // n, n


def atlas_uv_corners(c):
    """-> float32 [2, 3, 2] UV corners (texel units, cell-relative) of the even and the odd face of a cell"""
    return np.array([[(1, 1), (c - 3, 1), (1, c - 3)], [(c - 1, c - 1), (3, c - 1), (c - 1, 3)]], np.float32)


def atlas_owner(T, c, n, F):
    """-> int32 [T, T] owning face of each texel (-1 = none): Chebyshev distance < 1 from the face's UV triangle"""
    r, x = np.meshgrid(np.arange(T), np.arange(T), indexing="ij")
    px, py = x // c, r // c
    i, j = x - px * c, r - py * c
    cell = py * n + px
    valid = (px < n) & (py < n)
    a = valid & (i <= c - 3) & (j <= c - 3) & (i + j <= c - 2) & (2 * cell < F)
    b = valid & (i >= 2) & (j >= 2) & (i + j >= c) & (2 * cell + 1 < F)
    own = np.full((T, T), -1, np.int64)
    own[a] = 2 * cell[a]
    own[b] = 2 * cell[b] + 1
    return own.astype(np.int32)


def atlas_texels(v, f, T, c, n, bound):
    """-> (points float32 [T,T,3], owner int32 [T,T], vt float32 [3F,2]).  Each owned texel centre goes through its face's affine
    UV -> xyz map (gutter texels extrapolate slightly) and is clamped to [-bound, bound]; unowned texels get the point 0."""
    v = np.asarray(v, np.float32)
    f = np.asarray(f, np.int64)
    F = f.shape[0]
    owner = atlas_owner(T, c, n, F)
    r, x = np.nonzero(owner >= 0)
    o = owner[r, x].astype(np.int64)
    cell = o // 2
    odd = (o & 1) == 1
    li = (x - (cell % n) * c).astype(np.float32) + np.float32(0.5)
    lj = (r - (cell // n) * c).astype(np.float32) + np.float32(0.5)
    d = np.float32(c - 4)
    one, cm1 = np.float32(1), np.float32(c - 1)
    b1 = np.where(odd, (cm1 - li) / d, (li - one) / d).astype(np.float32)
    b2 = np.where(odd, (cm1 - lj) / d, (lj - one) / d).astype(np.float32)
    v0, v1, v2 = v[f[o, 0]], v[f[o, 1]], v[f[o, 2]]
    p = (v0 + b1[:, None] * (v1 - v0)) + b2[:, None] * (v2 - v0)
    p = np.minimum(np.maximum(p, np.float32(-bound)), np.float32(bound))
    points = np.zeros((T, T, 3), np.float32)
    points[r, x] = p
    uv = atlas_uv_corners(c)                                       # [2, 3, 2]
    fi = np.arange(F)
    origin = np.stack([(fi // 2) % n, (fi // 2) // n], axis=-1).astype(np.float32) * np.float32(c)
    vt = (origin[:, None, :] + uv[fi & 1]) / np.float32(T)           # [F, 3, 2]
    return points, owner, vt.reshape(-1, 2).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------------
# mesh checks shared by the tests
# ---------------------------------------------------------------------------------------------------------------------------
def directed_edges(faces):
    f = np.asarray(faces, np.int64)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def is_closed_oriented(faces):
    """every undirected edge in exactly two faces, traversed once in each direction"""
    e = directed_edges(faces)
    if len(e) == 0:
        return True
    key = e[:, 0] * (int(e.max()) + 1) + e[:, 1]
    rkey = e[:, 1] * (int(e.max()) + 1) + e[:, 0]
    u, cnt = np.unique(key, return_counts=True)
    if (cnt != 1).any():
        return False
    return bool(np.isin(rkey, u).all())


def euler_characteristic(verts, faces):
    e = directed_edges(faces)
    und = np.unique(np.sort(e, axis=1), axis=0)
    return len(verts) - len(und) + len(faces)


def signed_volume(verts, faces):
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)
