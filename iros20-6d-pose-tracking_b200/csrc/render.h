// Input A on the GPU: the object's CAD model rasterised at the previous pose into the 176 x 176 crop window (see render.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
namespace se3tn {
struct MeshDev {            // one CAD model in device memory (what vispy_renderer.py:108-129 uploads as vertex / index buffers)
    const float* pos;       // [nv][3] metres, object frame
    const float* nrm;       // [nv][3] unit normals
    const uint8_t* col;     // [nv][3] 8-bit colours
    const int* faces;       // [nf][3]
    int nv, nf;
};
struct RenderArgs {
    const double* poses;           // [n][16] object in OpenCV camera
    const double* object_width;    // [n] mm
    const int* mesh_ids;           // [n] or null (mesh 0)
    const MeshDev* meshes;         // device table indexed by mesh id
    int n_meshes;
    double fx, fy, cx, cy;
    uint8_t* projected;            // workspace [n][max_nv] projected vertices (render_projected_bytes_per_vertex() each)
    uint8_t* uniforms;             // workspace [n] per-track uniforms (render_uniform_bytes() each)
    int max_nv;                    // vertex count of the largest model
    int mode;                      // 0: vispy-style (lit, the crop window is the viewport); 1: pyrender-style (unlit full camera image vw x vh, then crop_bbox)
    int vw, vh;                    // mode 1: camera image size
    uint8_t* rgb;                  // [n][176][176][3], or null: depth only (the fit check of a track step)
    uint16_t* depth;               // [n][176][176] mm, 0 = background
    int32_t* tri = nullptr;        // [n][176][176] the triangle each pixel shows (depth's layout), -1 = background; or null
};
size_t render_uniform_bytes();
size_t render_projected_bytes_per_vertex();
// pdl = false: the projection starts only once the launch before it has completed (a step whose first kernel writes the poses,
// ids and widths that kernels after the render read before their griddepcontrol.wait).
cudaError_t launch_render(const RenderArgs& a, int n, cudaStream_t s, bool pdl = true);
// The visibility check of produce_train_pair_data.py:97-104 for n rows of one frame: each row's model rendered over the whole
// vh x vw camera image in the pyrender mode (nearest float32 window z per pixel into zmin, n x vh x vw words of scratch), then
// visible[i] = #(seg == class_ids[i]) and covered[i] = #(linearised depth > 0.1f).  class_ids, visible, covered device (n).
// Memsets + 3 launches; `a.mode` and `a.object_width` are ignored.
cudaError_t launch_coverage(RenderArgs a, int n, int max_nf, const uint8_t* seg, const int* class_ids, unsigned* zmin,
                            int* visible, int* covered, cudaStream_t s);
}  // namespace se3tn
