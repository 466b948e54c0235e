// keyframe_mesh_test.cpp -- the keyframe mesh facade (df::KeyframeMesher of df/dfk_mesh.h) against the C call it wraps,
// on two random keyframes of different sizes (one with every optional view, one with none):
//   Mesh(items, out)  equals dfk_keyframe_mesh_batch's rows, counts and uint16 depth for the same items
//   Item(...)         takes the cameras as the reference passes them: df::PinholeCamera-style objects and DfkCamera
//   the counts        fit the default capacities, and every triangle corner is a vertex of its item
// Build: see tests/cpp/keyframe_mesh.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "df/dfk_mesh.h"

#define EXPECT(c)                                                                       \
  do {                                                                                  \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

static void* dev_alloc(size_t bytes)
{
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) { std::puts("cudaMalloc failed"); std::exit(2); }
  cudaMemset(p, 0xAB, bytes);
  return p;
}

template <typename T>
static DfkImage upload(const std::vector<T>& host, int w, int h, int per_px)
{
  void* p = dev_alloc(host.size() * sizeof(T));
  cudaMemcpy(p, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice);
  return DfkImage{p, (size_t)w * per_px * sizeof(T), (uint32_t)w, (uint32_t)h};
}

template <typename T>
static std::vector<T> download(const void* p, size_t count)
{
  std::vector<T> v(count);
  cudaMemcpy(v.data(), p, count * sizeof(T), cudaMemcpyDeviceToHost);
  return v;
}

struct Cam {  // df::PinholeCamera<float>'s accessors
  DfkCamera c;
  float fx() const { return c.fx; }
  float fy() const { return c.fy; }
  float u0() const { return c.u0; }
  float v0() const { return c.v0; }
  float width() const { return c.width; }
  float height() const { return c.height; }
};

struct Outputs {
  df::KeyframeMeshOutput o;
  size_t v, t;
  Outputs(size_t v_rows, size_t t_rows, int n) : v(v_rows), t(t_rows)
  {
    o.positions = (float*)dev_alloc(12 * v);
    o.normals = (float*)dev_alloc(12 * v);
    o.pixels = (int32_t*)dev_alloc(4 * v);
    o.triangles = (int32_t*)dev_alloc(12 * t);
    o.counts = (int32_t*)dev_alloc(8 * (size_t)n);
  }
  std::vector<uint8_t> bytes() const
  {
    std::vector<uint8_t> b;
    for (auto [p, s] : {std::pair<const void*, size_t>{o.positions, 12 * v}, {o.normals, 12 * v}, {o.pixels, 4 * v},
                        {o.triangles, 12 * t}}) {
      const std::vector<uint8_t> x = download<uint8_t>(p, s);
      b.insert(b.end(), x.begin(), x.end());
    }
    return b;
  }
};

int main()
{
  std::mt19937 rng(7);
  std::uniform_real_distribution<float> depth(0.4f, 3.0f), logstd(-2.0f, 1.5f), vld(-0.2f, 1.0f);
  const int W0 = 96, H0 = 64, W1 = 70, H1 = 41;
  std::vector<float> d0(W0 * H0), s0(W0 * H0), v0(W0 * H0), d1(W1 * H1);
  std::vector<uint8_t> c0(3 * W0 * H0);
  for (float& x : d0) x = depth(rng);
  for (float& x : s0) x = logstd(rng);
  for (float& x : v0) x = vld(rng);
  for (uint8_t& x : c0) x = (uint8_t)(rng() & 255);
  for (float& x : d1) x = depth(rng);
  const Cam cam0{DfkCamera{80.0f, 81.0f, 47.5f, 31.5f, (float)W0, (float)H0}};
  const DfkCamera cam1{60.0f, 60.0f, 35.0f, 20.0f, (float)W1, (float)H1};
  const float pose0[7] = {0.1f, -0.2f, 0.05f, 0.9721f, 0.3f, -1.0f, 2.0f};
  const float pose1[7] = {0.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.0f};
  const DfkImage u16_a{dev_alloc(2 * W0 * H0), 2 * (size_t)W0, (uint32_t)W0, (uint32_t)H0};
  const DfkImage u16_b{dev_alloc(2 * W0 * H0), 2 * (size_t)W0, (uint32_t)W0, (uint32_t)H0};

  df::KeyframeMesher mesher;
  mesher.params().crop_pix = 4;
  const DfkImage dd0 = upload(d0, W0, H0, 1), ds0 = upload(s0, W0, H0, 1), dv0 = upload(v0, W0, H0, 1);
  const DfkImage dc0 = upload(c0, W0, H0, 3), dd1 = upload(d1, W1, H1, 1);
  std::vector<DfkKeyframeMeshItem> items{df::KeyframeMesher::Item(dd0, ds0, dv0, dc0, cam0, pose0, u16_a),
                                         df::KeyframeMesher::Item(dd1, DfkImage{}, DfkImage{}, DfkImage{}, cam1, pose1)};
  const std::vector<long long> vo = df::KeyframeMesher::VertexOffsets(items), to = df::KeyframeMesher::TriangleOffsets(items);
  EXPECT(vo.back() == W0 * H0 + W1 * H1 && to.back() == 2 * vo.back());
  Outputs a(vo.back(), to.back(), 2), b(vo.back(), to.back(), 2);
  mesher.Mesh(items, a.o);
  std::vector<DfkKeyframeMeshItem> items_c = items;
  items_c[0].depth_u16 = u16_b;
  const DfkKeyframeMeshParams p = mesher.params();
  EXPECT(dfk_keyframe_mesh_batch(mesher.handle(), items_c.data(), 2, 0, &p, b.o.positions, b.o.normals, nullptr,
                                 b.o.pixels, b.o.triangles, b.o.counts) == DFK_OK);
  EXPECT(cudaDeviceSynchronize() == cudaSuccess);
  EXPECT(a.bytes() == b.bytes());
  const std::vector<int32_t> ca = download<int32_t>(a.o.counts, 4), cb = download<int32_t>(b.o.counts, 4);
  EXPECT(ca == cb);
  EXPECT(download<uint16_t>(u16_a.ptr, W0 * H0) == download<uint16_t>(u16_b.ptr, W0 * H0));
  for (int i = 0; i < 2; ++i) {
    EXPECT(ca[2 * i] > 0 && ca[2 * i] <= items[i].vertex_capacity);
    EXPECT(ca[2 * i + 1] > 0 && ca[2 * i + 1] <= items[i].triangle_capacity);
    const std::vector<int32_t> tri = download<int32_t>(a.o.triangles + 3 * to[i], 3 * (size_t)ca[2 * i + 1]);
    for (int32_t k : tri) EXPECT(k >= 0 && k < ca[2 * i]);
  }
  std::printf("keyframe_mesh_test OK: counts (%d, %d) and (%d, %d)\n", ca[0], ca[1], ca[2], ca[3]);
  return 0;
}
