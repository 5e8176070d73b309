// C ABI over the reference checkout's header-only CDT (thirdparty/cdt), exactly as TrackPlane.cpp:717-723 drives it: float vertices
// inserted in the order given, super-triangle erased.  Test infrastructure: tests load the built oracle/_ref/libref_cdt.so.
#include "CDT.h"
#include <exception>
#include <vector>

extern "C" {
// xy[2n] floats; tri3 receives up to cap triangles (vertex indices).  Returns the triangle count, or -1 when CDT throws.
int ref_cdt_triangulate(int n, const float *xy, int cap, int *tri3) {
  try {
    std::vector<CDT::V2d<float>> v;
    for (int i = 0; i < n; i++)
      v.emplace_back(CDT::V2d<float>::make(xy[2 * i], xy[2 * i + 1]));
    CDT::Triangulation<float> cdt(CDT::VertexInsertionOrder::Enum::AsProvided);
    cdt.insertVertices(v);
    cdt.eraseSuperTriangle();
    const int nt = (int)cdt.triangles.size();
    for (int t = 0; t < nt && t < cap; t++)
      for (int j = 0; j < 3; j++)
        tri3[3 * t + j] = (int)cdt.triangles[t].vertices[j];
    return nt;
  } catch (const std::exception &) {
    return -1;
  }
}
}
