// fiesta_b200 -- surface meshes of the map: the triangle mesh of the boundary of what blocks at a clearance over a voxel box, with
// vertices placed on the records' exact distances.  Plain C++ shared by the kernels (fb_mesh.cu) and CPU tests
// (tests/cpp/mesh_test.cpp, g++).
//
// Definition (DESIGN.md §3.15).  Inputs: an inclusive box B = [lo, hi] (0 <= lo <= hi < grid size on every axis), a clearance r and
// flags (FIESTA_SEGMENT_*).  The result is a snapshot of the integrated records at the time of the call.
//   1. Blocking.  A voxel v of B blocks when fb_seg_blocks(g, rec, v, r, flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS, d) is true.  Voxels
//      outside B never block, the virtual layer one voxel outside each face of B included, so every mesh is closed and caps the box.
//   2. Distance.  v has a distance when it is in B and its record holds an obstacle that is not under an EXACT local-map reset (the
//      skeleton's "o(v) defined", fb_mesh_has_distance); d(v) = fb_record_distance of the record.
//   3. Extended box.  E = [lo - 1, hi] on every axis, (Bx+1)(By+1)(Bz+1) positions indexed
//      ((x-lo.x+1)*(By+1) + (y-lo.y+1))*(Bz+1) + (z-lo.z+1).  Cells and edges share this index space.
//   4. Crossing on a grid edge (u, w = u + e_a), u the lower endpoint, exactly one of them blocking: when both have a distance,
//      t = (r - d(u)) / (d(w) - d(u)) in fp64, each operation rounded on its own, so t is in [0, 1] (an end is reached when the
//      blocking endpoint's distance equals r); otherwise t = 0.5.  The crossing point is u + t e_a (fb_mesh_t).
//   5. Vertices.  Cell c in E has the corners c + {0,1}^3 and is active when its corners neither all block nor all fail to block.
//      Vertex ids are the ranks of the active cells in E-index order.  The position is the fp64 mean of the crossing points on the
//      cell's sign-changing edges, summed from 0.0 in a fixed order -- the 4 x-edges, then the 4 y-edges, then the 4 z-edges, each
//      axis' edges ordered lexicographically by the other two offsets (fb_mesh_cell_edge) -- and divided by (double)count; each
//      coordinate m becomes metres as ((m + 0.5) * resolution) + origin (Vox2Pos) and is rounded once to float32 (fb_mesh_vertex).
//   6. Faces.  One quad per sign-changing grid edge (v, v + e_a), v in E, a = x, y, z.  With (a, b, c) the cyclic triple (x,y,z),
//      (y,z,x) or (z,x,y), its corners are the cells q0 = v + (0,-1,-1), q1 = v + (0,0,-1), q2 = v, q3 = v + (0,-1,0) (offsets along
//      a, b, c), ordered q0 q1 q2 q3 when v blocks (normal +e_a) and q0 q3 q2 q1 otherwise: normals point from blocking to free
//      space (fb_mesh_quad).  The quad (p0 p1 p2 p3) in that order is split along p0-p2 when |p0-p2|^2 <= |p1-p3|^2 (fp64
//      differences and squares of the float32 positions, x, y and z summed in that order) into (p0,p1,p2), (p0,p2,p3), and
//      otherwise into (p1,p2,p3), (p1,p3,p0) (fb_mesh_split02, fb_mesh_tris).  Triangles are written in order of (v's E-index,
//      axis x, y, z), two per quad.
// Consequences: the mesh is combinatorially the boundary of the union of the blocking voxels' cubes (the cuberille surface, its
// vertices moved inside their cells) and is closed: every directed edge is matched by its reverse.  Blocking voxels that touch only
// along an edge or at a corner share the vertices there (non-manifold, still closed).  Clearance 0 puts the surface through obstacle
// voxel centres, 0.5 * resolution on the obstacle cubes' faces (every crossing is a midpoint), larger clearances on the inflated
// surface the planner queries avoid.  A clearance equal to a voxel's distance can give zero-area triangles; they are kept.  A vertex
// depends only on its cell's 8 corners, so the meshes of adjacent boxes agree bit for bit on the cells whose corners are real voxels
// of both boxes: a large map can be meshed in chunks.
#ifndef FB_MESH_H_
#define FB_MESH_H_
#include "fb_record.h"

// Vertex ranks are counted in uint32: an extended box of the largest grid, (2046 + 1) x (1024 + 1) x (1024 + 1) positions, has
// fewer than 2^32 of them.  Vertex ids are int32; a compute whose mesh would have more than 2^31 - 1 vertices (possible only for
// boxes of more than 2^31 - 1 extended positions, i.e. near the largest grid) fails with FIESTA_ERR_LIMIT.
static_assert(2047ull * 1025ull * 1025ull < (1ull << 32), "extended-box positions must fit the uint32 vertex ranks");

// Does a packed record give its voxel a distance?  (An obstacle, not under an EXACT local-map reset.)
FB_HD bool fb_mesh_has_distance(uint32_t c) {
  if (c & FB_DINF) return false;
  c &= FB_CODE_MASK;
  return c != FB_UNKNOWN && c != FB_INF;
}

// Crossing parameter on an edge from its lower endpoint u to its upper endpoint w, exactly one of them blocking.
FB_HD double fb_mesh_t(bool has_u, double du, bool has_w, double dw, double r) {
  if (!(has_u && has_w)) return 0.5;
  const double num = r - du;
  const double den = dw - du;
  return num / den;
}

// Corner k of a cell is the voxel c + ((k >> 2) & 1, (k >> 1) & 1, k & 1).  Cell edge e in 0..11, in the summation order: axis
// a = e / 4; the other two axes, in increasing order, take the offsets ((e >> 1) & 1, e & 1).  k0 / k1: its lower / upper corner.
FB_HD void fb_mesh_cell_edge(int e, int *a, int *k0, int *k1) {
  *a = e >> 2;
  const int p = *a == 0 ? 1 : 0, q = *a == 2 ? 1 : 2;
  int lo[3] = {0, 0, 0};
  lo[p] = (e >> 1) & 1;
  lo[q] = e & 1;
  *k0 = (lo[0] << 2) | (lo[1] << 1) | lo[2];
  *k1 = *k0 | (4 >> *a);
}

// The vertex of an active cell with lower corner c (grid voxel coordinates, lo - 1 allowed) from its 8 corners' blocking flags,
// distance flags and distances (index k as above).
FB_HD void fb_mesh_vertex(const int *c, const bool *blk, const bool *has, const double *d, double r, double res, const double *origin,
                          float *xyz) {
  double s[3] = {0.0, 0.0, 0.0};
  int n = 0;
  for (int e = 0; e < 12; ++e) {
    int a, k0, k1;
    fb_mesh_cell_edge(e, &a, &k0, &k1);
    if (blk[k0] == blk[k1]) continue;
    const double t = fb_mesh_t(has[k0], d[k0], has[k1], d[k1], r);
    for (int k = 0; k < 3; ++k) {
      const double u = (double)(c[k] + ((k0 >> (2 - k)) & 1));
      s[k] = s[k] + (k == a ? u + t : u);
    }
    ++n;
  }
  for (int k = 0; k < 3; ++k) {
    const double m = s[k] / (double)n;
    xyz[k] = (float)(((m + 0.5) * res) + origin[k]);
  }
}

// The four cells around the edge (v, v + e_a) as offsets from v, in the oriented order.
FB_HD void fb_mesh_quad(int a, bool v_blocks, int off[4][3]) {
  const int b = (a + 1) % 3, c = (a + 2) % 3;
  for (int i = 0; i < 4; ++i) {
    const int q = v_blocks ? i : (4 - i) & 3;                                 // q0 q1 q2 q3, or q0 q3 q2 q1
    off[i][a] = 0;
    off[i][b] = (q == 0 || q == 3) ? -1 : 0;
    off[i][c] = q < 2 ? -1 : 0;
  }
}

// The diagonal rule on the float32 positions of the quad's corners in oriented order: true splits along p0-p2.
FB_HD bool fb_mesh_split02(const float *p0, const float *p1, const float *p2, const float *p3) {
  double s02 = 0.0, s13 = 0.0;
  for (int k = 0; k < 3; ++k) {
    const double a = (double)p0[k] - (double)p2[k];
    const double b = (double)p1[k] - (double)p3[k];
    s02 = s02 + a * a;
    s13 = s13 + b * b;
  }
  return s02 <= s13;
}
// The quad's two triangles from its vertex ids q in oriented order.
FB_HD void fb_mesh_tris(const int32_t *q, bool split02, int32_t *out) {
  out[0] = split02 ? q[0] : q[1];
  out[1] = split02 ? q[1] : q[2];
  out[2] = split02 ? q[2] : q[3];
  out[3] = out[0];
  out[4] = out[2];
  out[5] = split02 ? q[3] : q[0];
}
#endif
