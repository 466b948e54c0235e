// dfk_mesh.h -- the keyframe renderer's geometry (gui/shaders/drawkf.geom) and SaveKeyframes' uint16 depth on top of
// dfk_keyframe_mesh_batch (include/dfk.h):
//   df::KeyframeMesher                     owns a handle and the renderer's parameters
//     .Item(dpt, std, vld, color, cam, pose_wk)   one keyframe's item from its fields (pyr_dpt / pyr_stdev / pyr_vld
//                                          level 0, color_img, pose_wk), capacities for every possible row
//     .Mesh(items, out)                    many keyframes in one call into the caller's device buffers
//     VertexOffsets / TriangleOffsets      where each item's rows start
// Views are DEVICE views the caller owns; a view with ptr = nullptr is absent.  Cameras are df::PinholeCamera<float>
// (accessors, as in the rest of the facade) or DfkCamera.
#ifndef DFK_MESH_H_
#define DFK_MESH_H_

#include <vector>

#include "dfk_facade.h"

namespace df
{

// The device outputs of a call (see dfk_keyframe_mesh_batch); only positions and counts are required
struct KeyframeMeshOutput {
  float* positions = nullptr;
  float* normals = nullptr;
  uint8_t* colors = nullptr;
  int32_t* pixels = nullptr;
  int32_t* triangles = nullptr;
  int32_t* counts = nullptr;
};

class KeyframeMesher
{
public:
  // the visualizer's defaults (gui/visualizer.cpp:657-661)
  static DfkKeyframeMeshParams DefaultParams() { return DfkKeyframeMeshParams{4.2f, 0.0f, 20, 0}; }

  explicit KeyframeMesher(DfkKeyframeMeshParams params = DefaultParams()) : params_(params), h_(detail::MakeHandle()) {}

  DfkHandle handle() const { return h_.get(); }
  void SetStream(void* stream) { detail::Check(h_.get(), dfk_set_stream(h_.get(), stream)); }
  DfkKeyframeMeshParams& params() { return params_; }

  // One keyframe from its depth; std, vld, color and depth_u16 may be {} (absent).  The capacities allow every vertex
  // (W H) and every triangle (2 W H); a caller that knows its counts from an earlier call may set smaller ones.
  template <typename CamT>
  static DfkKeyframeMeshItem Item(const DfkImage& dpt, const DfkImage& std, const DfkImage& vld, const DfkImage& color,
                                  const CamT& camera, const float pose_wk[7], const DfkImage& depth_u16 = DfkImage{})
  {
    DfkKeyframeMeshItem it{};
    it.dpt = dpt;
    it.std = std;
    it.valid = vld;
    it.color = color;
    it.cam = detail::Cam(camera);
    for (int k = 0; k < 7; ++k) it.pose_wk[k] = pose_wk[k];
    const long long px = static_cast<long long>(it.cam.width) * static_cast<long long>(it.cam.height);
    it.vertex_capacity = static_cast<int32_t>(px);
    it.triangle_capacity = static_cast<int32_t>(2 * px);
    it.depth_u16 = depth_u16;
    return it;
  }

  // many keyframes in one call; code_size is needed only by items that decode their depth
  void Mesh(const std::vector<DfkKeyframeMeshItem>& items, const KeyframeMeshOutput& out, int code_size = 0)
  {
    detail::Check(h_.get(), dfk_keyframe_mesh_batch(h_.get(), items.data(), static_cast<int>(items.size()), code_size,
                                                    &params_, out.positions, out.normals, out.colors, out.pixels,
                                                    out.triangles, out.counts));
  }

  // the first vertex / triangle row of each item, and the rows of the call at the end (n + 1 entries)
  static std::vector<long long> VertexOffsets(const std::vector<DfkKeyframeMeshItem>& items)
  {
    std::vector<long long> o{0};
    for (const DfkKeyframeMeshItem& it : items) o.push_back(o.back() + it.vertex_capacity);
    return o;
  }
  static std::vector<long long> TriangleOffsets(const std::vector<DfkKeyframeMeshItem>& items)
  {
    std::vector<long long> o{0};
    for (const DfkKeyframeMeshItem& it : items) o.push_back(o.back() + it.triangle_capacity);
    return o;
  }

private:
  DfkKeyframeMeshParams params_;
  detail::HandlePtr h_;
};

}  // namespace df

#endif  // DFK_MESH_H_
