// TEST HARNESS ONLY — CPU lane-emulation of the vertex-normal kernels (mb2_character_vertex_normals*_device), part of
// tests/emu/libmb2_emu.so.
//
// The face tables are made by the library's own makeMeshFaces; the __host__ __device__ building blocks of ik_device.cuh then run in the
// kernels' order for each vertex: its corner list in order with faceNormal, then normalizeClamped (vertexNormalKernel); for the backward
// normalGradient into h (the first pass), then per corner G_f = h_i0 + h_i1 + h_i2 and cornerGradient (vertexNormalGradKernel). An
// instance's sums do not depend on the kernels' tile of instances, so one instance at a time is what every tile computes. It is not part
// of the product library and nothing in momentum_b200/ loads it.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "emu_error.h"

using namespace mb2;

namespace {
int make(int32_t V, int32_t F, const int32_t* faces, HostMeshFaces& m) {
  g_emuErr = makeMeshFaces(V, F, faces, m);
  return g_emuErr.empty() ? MB2_OK : MB2_ERR_INVALID_ARGUMENT;
}

// n_v of one instance, over the vertex's corner list in order
F3 vertexSum(const HostMeshFaces& m, const float* x, int v) {
  F3 n = f3(0.f, 0.f, 0.f);
  for (int c = m.vertStart[v]; c < m.vertStart[v + 1]; ++c) {
    const int* f = m.faces.data() + (m.vertCorner[c] / 3) * 3;
    n = n + faceNormal(ld3(x + 3 * f[0]), ld3(x + 3 * f[1]), ld3(x + 3 * f[2]));
  }
  return n;
}
} // namespace

// makeMeshFaces alone: the vertex -> corner table (vertStart [V+1], vertCorner [3F]) it builds, or its message
extern "C" int emu_mesh_faces_tables(int32_t V, int32_t F, const int32_t* faces, int32_t* vertStart, int32_t* vertCorner) {
  HostMeshFaces m;
  if (make(V, F, faces, m) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  std::copy(m.vertStart.begin(), m.vertStart.end(), vertStart);
  std::copy(m.vertCorner.begin(), m.vertCorner.end(), vertCorner);
  return MB2_OK;
}

// positions [B][V][3] -> normals [B][V][3]
extern "C" int emu_vertex_normals(int32_t V, int32_t F, const int32_t* faces, int32_t batch, const float* positions, float* normals) {
  HostMeshFaces m;
  if (make(V, F, faces, m) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  for (int b = 0; b < batch; ++b) {
    const float* x = positions + size_t(b) * V * 3;
    for (int v = 0; v < V; ++v) {
      const F3 r = normalizeClamped(vertexSum(m, x, v));
      float* o = normals + (size_t(b) * V + v) * 3;
      o[0] = r.x; o[1] = r.y; o[2] = r.z;
    }
  }
  return MB2_OK;
}

// the backward: gradPositions [B][V][3] from gradNormals [B][V][3]
extern "C" int emu_vertex_normals_backward(int32_t V, int32_t F, const int32_t* faces, int32_t batch, const float* positions, const float* gradNormals,
                                           float* gradPositions) {
  HostMeshFaces m;
  if (make(V, F, faces, m) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  std::vector<float> h(size_t(V) * 3);
  for (int b = 0; b < batch; ++b) {
    const float* x = positions + size_t(b) * V * 3;
    for (int v = 0; v < V; ++v) { // vertexNormalKernel<true>
      const F3 r = normalGradient(vertexSum(m, x, v), ld3(gradNormals + (size_t(b) * V + v) * 3));
      h[3 * v] = r.x; h[3 * v + 1] = r.y; h[3 * v + 2] = r.z;
    }
    for (int v = 0; v < V; ++v) { // vertexNormalGradKernel
      F3 g = f3(0.f, 0.f, 0.f);
      for (int c = m.vertStart[v]; c < m.vertStart[v + 1]; ++c) {
        const int fc = m.vertCorner[c], k = fc % 3;
        const int* f = m.faces.data() + (fc - k);
        const F3 G = ld3(h.data() + 3 * f[0]) + ld3(h.data() + 3 * f[1]) + ld3(h.data() + 3 * f[2]);
        g = g + cornerGradient(ld3(x + 3 * f[(k + 1) % 3]), ld3(x + 3 * f[(k + 2) % 3]), G);
      }
      float* o = gradPositions + (size_t(b) * V + v) * 3;
      o[0] = g.x; o[1] = g.y; o[2] = g.z;
    }
  }
  return MB2_OK;
}
