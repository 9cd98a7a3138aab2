// GaussianSplatRenderer.hpp -- header-only C++ host mirror of the reference's C# component
// (package/Runtime/GaussianSplatRenderer.cs) over the C ABI in include/gsplat_b200.h.
// The reference's host language (C# / Unity) has no toolchain in this image; C++ is the compiled
// host language used instead.  Same member names and call order as the C# class for the hot path;
// errors never throw: like the reference (:361-369,:655) a failed call logs and returns false.
#pragma once
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/gsplat_b200.h"

namespace GaussianSplatting {

struct Matrix4x4 { float m[16]; };  // column-major, like UnityEngine.Matrix4x4

struct CameraState {               // what the C# code reads from UnityEngine.Camera
  Matrix4x4 worldToCameraMatrix;   // :586
  Matrix4x4 gpuProjectionMatrix;   // GL.GetGPUProjectionMatrix(cam.projectionMatrix, true)
  float pixelWidth, pixelHeight;   // :589-591
  float position[3];               // :592
};

// An image that is a 2-D CUDA array (GS_MEM_ARRAY): `array` is the cudaArray_t of RGBA16F / RGBA32F texels, created with
// cudaArraySurfaceLoadStore -- e.g. the render texture a graphics-interop plugin imported (cudaExternalMemoryGetMappedMipmappedArray,
// level 0).  It is rendered into / composited onto in place.
inline GsImage ArrayImage(void *array, uint32_t width, uint32_t height, uint32_t format = GS_PIX_RGBA16F) {
  GsImage im;
  std::memset(&im, 0, sizeof(im));
  im.data = array;
  im.width = width;
  im.height = height;
  im.row_pitch_bytes = 0;
  im.format = format;
  im.memory = GS_MEM_ARRAY;
  return im;
}

// An image that is one layer of a layered CUDA array (GS_MEM_ARRAY_LAYER), e.g. one eye of an XR eye-texture array or one face of
// a cube map, created with cudaArrayLayered | cudaArraySurfaceLoadStore.  The image points to `desc`, which must outlive every
// call the image is passed to.
inline GsImage ArrayLayerImage(GsArrayLayer *desc, uint32_t width, uint32_t height, uint32_t format = GS_PIX_RGBA16F) {
  GsImage im = ArrayImage(desc, width, height, format);
  im.memory = GS_MEM_ARRAY_LAYER;
  return im;
}

// An image that is a width x height rectangle of a 2-D CUDA array or of one layer of a layered one (GS_MEM_ARRAY_RECT): pixel
// (px, py) is texel (desc->x + px, desc->y + py).  E.g. a camera's part of an HDRP render target allocated larger than the camera
// (desc = {array, 0, 0, 0, 0}, width x height the camera's scaled pixel size), or one view's tile of an atlas.  The image points
// to `desc`, which must outlive every call the image is passed to.
inline GsImage ArrayRectImage(GsArrayRect *desc, uint32_t width, uint32_t height, uint32_t format = GS_PIX_RGBA16F) {
  GsImage im = ArrayImage(desc, width, height, format);
  im.memory = GS_MEM_ARRAY_RECT;
  return im;
}

// A camera target of packed B10G11R11_UFLOAT texels (GS_PIX_B10G11R11_UFLOAT: the HDR colour buffer of URP and HDRP cameras,
// accepted as a camera target only) in host or device memory (`memory`): one uint32 per pixel, rows `row_pitch_bytes` apart
// (0: tightly packed).  Such a colour buffer imported as a CUDA array (one 32-bit unsigned channel) is ArrayImage /
// ArrayLayerImage / ArrayRectImage with format GS_PIX_B10G11R11_UFLOAT.
inline GsImage PackedCameraTarget(void *data, uint32_t width, uint32_t height, uint32_t memory, uint32_t row_pitch_bytes = 0) {
  GsImage im;
  std::memset(&im, 0, sizeof(im));
  im.data = data;
  im.width = width;
  im.height = height;
  im.row_pitch_bytes = row_pitch_bytes;
  im.format = GS_PIX_B10G11R11_UFLOAT;
  im.memory = memory;
  return im;
}

// A camera target of R8G8B8A8_SRGB texels (GS_PIX_R8G8B8A8_SRGB: the colour buffer of an LDR camera in a linear-colour-space
// project, accepted as a camera target only) in host or device memory (`memory`): four bytes R, G, B, A per pixel, rows
// `row_pitch_bytes` apart (0: tightly packed).  Such a colour buffer imported as a CUDA array (four 8-bit unsigned channels) is
// ArrayImage / ArrayLayerImage / ArrayRectImage with format GS_PIX_R8G8B8A8_SRGB.
inline GsImage Srgb8CameraTarget(void *data, uint32_t width, uint32_t height, uint32_t memory, uint32_t row_pitch_bytes = 0) {
  GsImage im = PackedCameraTarget(data, width, height, memory, row_pitch_bytes);
  im.format = GS_PIX_R8G8B8A8_SRGB;
  return im;
}

// The payload of GS_UNITY_EVENT_FRAME_CAMERAS (GaussianSplatRenderer::FillFrameCamerasEvent) and the arrays it points to.
// `event` points into this object: keep it alive and unmoved until the event has run, and with it the renderers (their
// cutouts), the host images and the GsArrayLayer / GsArrayRect descriptors the images point to.
struct UnityFrameCamerasEvent {
  GsUnityFrameCamerasEvent event{};
  std::vector<uint32_t> counts;
  std::vector<GsAsset *> assets;
  std::vector<GsFrameParams> fps;
  std::vector<int32_t> doSort;
  std::vector<GsImage> rts, cameraTargets;   // by value; data == nullptr: none
};

// The payload of GS_UNITY_EVENT_GROUP_FRAME_OBJECTS (GaussianSplatRendererGroup::FillFrameObjectsEvent) and its arrays, under
// the same rule.
struct UnityGroupFrameObjectsEvent {
  GsUnityGroupFrameObjectsEvent event{};
  std::vector<GsAsset *> assets;
  std::vector<GsFrameParams> fps;
  std::vector<int32_t> doSort;
  std::vector<GsImage> rts, cameraTargets;   // by value, one per local member; data == nullptr: none
};

class GaussianSplatRenderer {
 public:
  // serialized knobs, :225-251
  float m_SplatScale = 1.0f, m_OpacityScale = 1.0f;
  int m_SHOrder = 3;
  bool m_SHOnly = false;
  int m_SortNthFrame = 1;
  int m_RenderOrder = 0;   // :236, higher values draw first
  Matrix4x4 localToWorldMatrix{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};
  Matrix4x4 worldToLocalMatrix{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};
  std::vector<GsCutout> m_Cutouts;
  // The camera's depth buffer the splats are depth-tested against (GsFrameParams.scene_depth), width x height float32 in
  // reversed Z, or nullptr.  sceneDepthMemory is its GsMemory (scene_depth_on_device): GS_MEM_HOST, GS_MEM_DEVICE, GS_MEM_ARRAY
  // (sceneDepth is a cudaArray_t of one float32 channel), GS_MEM_ARRAY_LAYER (SetSceneDepthLayer) or GS_MEM_ARRAY_RECT
  // (SetSceneDepthRect).
  const float *sceneDepth = nullptr;
  uint32_t sceneDepthMemory = GS_MEM_HOST;
  // The depth is one layer of a layered float32 CUDA array (e.g. one eye of an XR eye-depth array); `desc` must outlive every
  // frame drawn with it.
  void SetSceneDepthLayer(const GsArrayLayer *desc) {
    sceneDepth = reinterpret_cast<const float *>(desc);
    sceneDepthMemory = GS_MEM_ARRAY_LAYER;
  }
  // The depth is the width x height rectangle at (desc->x, desc->y) of a 2-D or layered float32 CUDA array (e.g. the camera's
  // part of an HDRP depth texture allocated larger than the camera); `desc` must outlive every frame drawn with it.
  void SetSceneDepthRect(const GsArrayRect *desc) {
    sceneDepth = reinterpret_cast<const float *>(desc);
    sceneDepthMemory = GS_MEM_ARRAY_RECT;
  }
  GsRenderOptions options{};

  ~GaussianSplatRenderer() { OnDisable(); }

  // OnEnable -> CreateResourcesForAsset, :373-445,:475
  bool OnEnable(const GsAssetDesc &asset, int cudaDevice = 0, void *stream = nullptr) {
    OnDisable();
    if (!ok(gs_create(cudaDevice, stream, &m_Ctx))) return false;
    m_OwnsCtx = true;
    if (!ok(gs_asset_upload(m_Ctx, &asset, &m_Asset))) return false;
    m_FrameCounter = 0;
    return true;
  }
  // The same on the context of another renderer (which must outlive this one): the splat objects of one camera share a
  // context so that SortAndRenderSplatsMulti draws them in one call.
  bool OnEnable(const GsAssetDesc &asset, GsContext *sharedContext) {
    OnDisable();
    if (!sharedContext) return false;
    m_Ctx = sharedContext;
    if (!ok(gs_asset_upload(m_Ctx, &asset, &m_Asset))) return false;
    m_FrameCounter = 0;
    return true;
  }
  // OnEnable of a renderer whose m_Asset `source` (enabled) already has: an instance of its asset (gs_asset_instance) on
  // source's context -- the blobs stay one copy in HBM, the draw order is this renderer's own.  The blobs outlive whichever
  // renderer is disabled first; the context must outlive this renderer, as for OnEnable(asset, sharedContext).
  bool CreateInstanceOf(const GaussianSplatRenderer &source) {
    OnDisable();
    if (!source.HasValidRenderSetup()) return false;
    m_Ctx = source.m_Ctx;
    if (!ok(gs_asset_instance(source.m_Asset, &m_Asset))) return false;
    m_FrameCounter = 0;
    return true;
  }
  void OnDisable() {  // :533-577
    if (m_Asset) gs_asset_destroy(m_Asset);
    if (m_Ctx && m_OwnsCtx) gs_destroy(m_Ctx);
    m_Asset = nullptr;
    m_Ctx = nullptr;
    m_OwnsCtx = false;
  }
  bool HasValidRenderSetup() const { return m_Ctx && m_Asset; }                           // :369
  bool SortPoints(const CameraState &cam) { GsFrameParams fp = params(cam); return ok(gs_sort(m_Ctx, m_Asset, &fp)); }          // :612
  bool CalcViewData(const CameraState &cam) { GsFrameParams fp = params(cam); return ok(gs_calc_view(m_Ctx, m_Asset, &fp)); }   // :579
  bool DrawSplats(const CameraState &cam, GsImage *rt) { GsFrameParams fp = params(cam); return ok(gs_render(m_Ctx, m_Asset, &fp, &options, rt)); }  // :165
  bool Composite(const GsImage *rt, GsImage *cameraTarget) { return ok(gs_composite(m_Ctx, rt, cameraTarget)); }               // :206-210
  // one renderer's share of GaussianSplatRenderSystem.SortAndRenderSplats, :108-169
  bool SortAndRenderSplats(const CameraState &cam, GsImage *rt, GsImage *cameraTarget = nullptr) {
    const int doSort = (m_FrameCounter % (m_SortNthFrame > 0 ? m_SortNthFrame : 1)) == 0;  // :120-121
    ++m_FrameCounter;
    GsFrameParams fp = params(cam);
    return ok(gs_frame(m_Ctx, m_Asset, &fp, &options, doSort, rt, cameraTarget));
  }
  // GaussianSplatRenderSystem.SortAndRenderSplats for one camera (:73-105,108-169,187-211): `renderers` (all on one context)
  // drawn in GatherSplatsForCamera order into one target, cleared once, then composited onto cameraTarget (may be nullptr) --
  // one gs_frame_objects call.  options (blend mode, asynchronous read-back) are the first drawn renderer's.
  static bool SortAndRenderSplatsMulti(const CameraState &cam, std::vector<GaussianSplatRenderer *> renderers, GsImage *rt,
                                       GsImage *cameraTarget = nullptr) {
    auto depth = [&](const GaussianSplatRenderer *r) {   // camera-space z of the object's position, +z forward
      const float *v = cam.worldToCameraMatrix.m, *p = r->localToWorldMatrix.m + 12;
      return -(v[2] * p[0] + v[6] * p[1] + v[10] * p[2] + v[14]);
    };
    if (renderers.empty()) return true;   // no active splat object: OnPreCullCamera draws nothing
    for (const GaussianSplatRenderer *r : renderers)   // checked before any renderer's frame counter moves
      if (!r || !r->HasValidRenderSetup() || r->m_Ctx != renderers[0]->m_Ctx) return false;
    std::stable_sort(renderers.begin(), renderers.end(), [&](const GaussianSplatRenderer *a, const GaussianSplatRenderer *b) {
      if (a->m_RenderOrder != b->m_RenderOrder) return a->m_RenderOrder > b->m_RenderOrder;
      return depth(a) < depth(b);
    });
    std::vector<GsAsset *> assets;
    std::vector<GsFrameParams> fps;
    std::vector<int32_t> doSort;
    for (GaussianSplatRenderer *r : renderers) {
      assets.push_back(r->m_Asset);
      fps.push_back(r->params(cam));
      doSort.push_back((r->m_FrameCounter % (r->m_SortNthFrame > 0 ? r->m_SortNthFrame : 1)) == 0);   // :120-121
      ++r->m_FrameCounter;
    }
    GsRenderOptions opt = renderers[0]->options;
    opt.flags &= ~(uint32_t)GS_FLAG_LOAD_RT;
    return renderers[0]->ok(gs_frame_objects(renderers[0]->m_Ctx, (uint32_t)renderers.size(), assets.data(), fps.data(), doSort.data(),
                                             &opt, rt, cameraTarget));
  }
  // The camera loop of GaussianSplatRenderSystem (OnPreCullCamera, :187-211): SortAndRenderSplatsMulti for cams[c] into rts[c] /
  // cameraTargets[c] (either may be nullptr, not both), one camera after the other.  Every renderer is gathered per camera
  // (GatherSplatsForCamera, :73-105) and its frame counter advances once per camera (:120-122).  All renderers share one
  // context.  When they also share their options (GS_FLAG_LOAD_RT aside) and none asks for GS_FLAG_ASYNC_READBACK, this is one
  // gs_frame_cameras call; otherwise it is that loop, SortAndRenderSplatsMulti per camera, as the Python mirror does.  A
  // renderer listed twice or a camera without any image returns false before any frame counter moves; what only the library
  // checks (screen and image sizes) returns false after they moved, as SortAndRenderSplatsMulti does.
  static bool SortAndRenderSplatsCameras(const std::vector<CameraState> &cams, const std::vector<GaussianSplatRenderer *> &renderers,
                                         const std::vector<GsImage *> &rts, const std::vector<GsImage *> &cameraTargets) {
    bool oneCall = false;
    if (!CheckCameras(cams, renderers, rts, cameraTargets, &oneCall)) return false;
    if (renderers.empty()) return true;
    if (!oneCall) {
      for (size_t c = 0; c < cams.size(); ++c)
        if (!SortAndRenderSplatsMulti(cams[c], renderers, rts[c], cameraTargets[c])) return false;
      return true;
    }
    std::vector<uint32_t> counts;
    std::vector<GsAsset *> assets;
    std::vector<GsFrameParams> fps;
    std::vector<int32_t> doSort;
    GaussianSplatRenderer *first = GatherCameras(cams, renderers, counts, assets, fps, doSort);
    if (!first) return true;   // no camera
    GsRenderOptions opt = first->options;
    opt.flags &= ~(uint32_t)GS_FLAG_LOAD_RT;
    return first->ok(gs_frame_cameras(first->m_Ctx, (uint32_t)counts.size(), counts.data(), assets.data(), fps.data(), doSort.data(), &opt,
                                      rts.data(), cameraTargets.data()));
  }
  // The render-thread event of SortAndRenderSplatsCameras' one call: fills *out with the payload of
  // GS_UNITY_EVENT_FRAME_CAMERAS (status GS_ERR_NOT_READY) for CommandBuffer.IssuePluginEventAndData, with the same checks,
  // GatherSplatsForCamera order and frame-counter steps, and the images copied by value.  Returns false, with no frame counter
  // moved, where SortAndRenderSplatsCameras would return false before drawing, where it would draw nothing (no renderer or no
  // camera), and where the renderers' options make it a loop of calls, which no one event carries.
  static bool FillFrameCamerasEvent(const std::vector<CameraState> &cams, const std::vector<GaussianSplatRenderer *> &renderers,
                                    const std::vector<GsImage *> &rts, const std::vector<GsImage *> &cameraTargets, UnityFrameCamerasEvent *out) {
    bool oneCall = false;
    if (!out || !CheckCameras(cams, renderers, rts, cameraTargets, &oneCall) || !oneCall || renderers.empty() || cams.empty()) return false;
    GaussianSplatRenderer *first = GatherCameras(cams, renderers, out->counts, out->assets, out->fps, out->doSort);
    out->rts.assign(cams.size(), GsImage{});
    out->cameraTargets.assign(cams.size(), GsImage{});
    for (size_t c = 0; c < cams.size(); ++c) {
      if (rts[c]) out->rts[c] = *rts[c];
      if (cameraTargets[c]) out->cameraTargets[c] = *cameraTargets[c];
    }
    GsUnityFrameCamerasEvent &ev = out->event;
    std::memset(&ev, 0, sizeof(ev));
    ev.ctx = first->m_Ctx;
    ev.camera_count = (uint32_t)out->counts.size();
    ev.object_counts = out->counts.data();
    ev.assets = out->assets.data();
    ev.fps = out->fps.data();
    ev.do_sort = out->doSort.data();
    ev.options = first->options;
    ev.options.flags &= ~(uint32_t)GS_FLAG_LOAD_RT;
    ev.rts = out->rts.data();
    ev.camera_targets = out->cameraTargets.data();
    ev.status = GS_ERR_NOT_READY;
    return true;
  }
  bool Sync() { return ok(gs_sync(m_Ctx)); }
  // EditExportData, R/GaussianSplatRenderer.cs:936-958: n x 62 floats (the .ply attribute record), cut splats marked by nor = 1
  bool EditExportData(float *dstRecords, bool bakeTransform = false) {
    return ok(gs_export_splats(m_Ctx, m_Asset, m_Cutouts.empty() ? nullptr : m_Cutouts.data(), (uint32_t)m_Cutouts.size(), bakeTransform ? 1u : 0u,
                               dstRecords));
  }
  GsContext *context() const { return m_Ctx; }
  GsAsset *asset() const { return m_Asset; }

 private:
  // What SortAndRenderSplatsCameras checks before any frame counter moves.  *oneCall: the renderers share their options
  // (GS_FLAG_LOAD_RT aside) and none asks for GS_FLAG_ASYNC_READBACK, so that one gs_frame_cameras call draws every camera.
  static bool CheckCameras(const std::vector<CameraState> &cams, const std::vector<GaussianSplatRenderer *> &renderers,
                           const std::vector<GsImage *> &rts, const std::vector<GsImage *> &cameraTargets, bool *oneCall) {
    *oneCall = true;
    if (rts.size() != cams.size() || cameraTargets.size() != cams.size()) return false;
    if (renderers.empty()) return true;
    for (const GaussianSplatRenderer *r : renderers)   // checked before any renderer's frame counter moves
      if (!r || !r->HasValidRenderSetup() || r->m_Ctx != renderers[0]->m_Ctx) return false;
    {
      std::vector<const GaussianSplatRenderer *> sorted(renderers.begin(), renderers.end());
      std::sort(sorted.begin(), sorted.end());
      if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) return false;
    }
    for (size_t c = 0; c < cams.size(); ++c)
      if (!rts[c] && !cameraTargets[c]) return false;
    auto same = [](const GsRenderOptions &a, const GsRenderOptions &b) {
      return a.blend_mode == b.blend_mode && a.band_packed == b.band_packed && a.partition_index == b.partition_index &&
             a.partition_count == b.partition_count && a.band_rows == b.band_rows && a.row_begin == b.row_begin && a.row_end == b.row_end &&
             ((a.flags ^ b.flags) & ~(uint32_t)GS_FLAG_LOAD_RT) == 0 && !(a.flags & GS_FLAG_ASYNC_READBACK);
    };
    for (const GaussianSplatRenderer *r : renderers) *oneCall = *oneCall && same(r->options, renderers[0]->options);
    return true;
  }
  // gs_frame_cameras' per-object arguments: every camera's renderers in GatherSplatsForCamera order (:73-105), camera after
  // camera, each renderer's frame counter advanced once per camera (:120-122).  Returns the first renderer drawn (nullptr: no
  // camera).
  static GaussianSplatRenderer *GatherCameras(const std::vector<CameraState> &cams, const std::vector<GaussianSplatRenderer *> &renderers,
                                              std::vector<uint32_t> &counts, std::vector<GsAsset *> &assets, std::vector<GsFrameParams> &fps,
                                              std::vector<int32_t> &doSort) {
    counts.clear(); assets.clear(); fps.clear(); doSort.clear();
    GaussianSplatRenderer *first = nullptr;
    for (size_t c = 0; c < cams.size(); ++c) {
      const CameraState &cam = cams[c];
      auto depth = [&](const GaussianSplatRenderer *r) {   // camera-space z of the object's position, +z forward
        const float *v = cam.worldToCameraMatrix.m, *p = r->localToWorldMatrix.m + 12;
        return -(v[2] * p[0] + v[6] * p[1] + v[10] * p[2] + v[14]);
      };
      std::vector<GaussianSplatRenderer *> order = renderers;
      std::stable_sort(order.begin(), order.end(), [&](const GaussianSplatRenderer *a, const GaussianSplatRenderer *b) {
        if (a->m_RenderOrder != b->m_RenderOrder) return a->m_RenderOrder > b->m_RenderOrder;
        return depth(a) < depth(b);
      });
      if (!first) first = order[0];
      counts.push_back((uint32_t)order.size());
      for (GaussianSplatRenderer *r : order) {
        assets.push_back(r->m_Asset);
        fps.push_back(r->params(cam));
        doSort.push_back((r->m_FrameCounter % (r->m_SortNthFrame > 0 ? r->m_SortNthFrame : 1)) == 0);   // :120-121
        ++r->m_FrameCounter;
      }
    }
    return first;
  }
  GsFrameParams params(const CameraState &cam) const {  // CalcViewData / SortPoints uniform binding, :586-606,:617-631
    GsFrameParams fp;
    std::memset(&fp, 0, sizeof(fp));
    std::memcpy(fp.mat_object_to_world, localToWorldMatrix.m, 64);
    std::memcpy(fp.mat_world_to_object, worldToLocalMatrix.m, 64);
    std::memcpy(fp.mat_view, cam.worldToCameraMatrix.m, 64);
    std::memcpy(fp.mat_proj_gpu, cam.gpuProjectionMatrix.m, 64);
    fp.screen_w = cam.pixelWidth;
    fp.screen_h = cam.pixelHeight;
    std::memcpy(fp.cam_pos_world, cam.position, 12);
    fp.splat_scale = m_SplatScale;
    fp.opacity_scale = m_OpacityScale;
    fp.sh_order = (uint32_t)m_SHOrder;
    fp.sh_only = m_SHOnly ? 1u : 0u;
    fp.cutouts = m_Cutouts.empty() ? nullptr : m_Cutouts.data();
    fp.cutout_count = (uint32_t)m_Cutouts.size();
    fp.scene_depth = sceneDepth;
    fp.scene_depth_on_device = sceneDepthMemory;
    return fp;
  }
  bool ok(int rc) const {
    if (rc == GS_OK) return true;
    std::fprintf(stderr, "GaussianSplatRenderer: %s (%d)\n", gs_last_error(m_Ctx), rc);  // Debug.LogError + skip
    return false;
  }
  GsContext *m_Ctx = nullptr;
  bool m_OwnsCtx = false;
  GsAsset *m_Asset = nullptr;
  int m_FrameCounter = 0;
};

// One splat object on a group: the renderer's knobs and its asset on every local member.  The group itself is one
// (GaussianSplatRendererGroup derives from it); AddObject makes more.
struct GaussianSplatGroupObject {
  float m_SplatScale = 1.0f, m_OpacityScale = 1.0f;
  int m_SHOrder = 3;
  bool m_SHOnly = false;
  int m_SortNthFrame = 1;
  int m_RenderOrder = 0;   // :236, higher values draw first
  Matrix4x4 localToWorldMatrix{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};
  Matrix4x4 worldToLocalMatrix{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};
  std::vector<GsCutout> m_Cutouts;
  const uint32_t *deletedBits = nullptr, *selectedBits = nullptr;   // host, ceil(N/32) words, or nullptr
  const float *sceneDepth = nullptr;                                 // host, width x height, or nullptr
  int m_FrameCounter = 0;
  std::vector<GsAsset *> m_Assets;                                   // [local member]

  GsFrameParams params(const CameraState &cam) const {
    GsFrameParams fp;
    std::memset(&fp, 0, sizeof(fp));
    std::memcpy(fp.mat_object_to_world, localToWorldMatrix.m, 64);
    std::memcpy(fp.mat_world_to_object, worldToLocalMatrix.m, 64);
    std::memcpy(fp.mat_view, cam.worldToCameraMatrix.m, 64);
    std::memcpy(fp.mat_proj_gpu, cam.gpuProjectionMatrix.m, 64);
    fp.screen_w = cam.pixelWidth;
    fp.screen_h = cam.pixelHeight;
    std::memcpy(fp.cam_pos_world, cam.position, 12);
    fp.splat_scale = m_SplatScale;
    fp.opacity_scale = m_OpacityScale;
    fp.sh_order = (uint32_t)m_SHOrder;
    fp.sh_only = m_SHOnly ? 1u : 0u;
    fp.cutouts = m_Cutouts.empty() ? nullptr : m_Cutouts.data();
    fp.cutout_count = (uint32_t)m_Cutouts.size();
    fp.deleted_bits = deletedBits;
    fp.selected_bits = selectedBits;
    fp.scene_depth = sceneDepth;
    return fp;
  }
  int nextDoSort() {   // :120-121
    const int doSort = (m_FrameCounter % (m_SortNthFrame > 0 ? m_SortNthFrame : 1)) == 0;
    ++m_FrameCounter;
    return doSort;
  }
};

// The same renderer on several GPUs of one box, one process driving all of them (gs_group_create / gs_group_frame):
// identical knobs; every non-null image receives the complete frame, bit-identical to what one GPU renders.
class GaussianSplatRendererGroup : public GaussianSplatGroupObject {
 public:
  GsRenderOptions options{};

  ~GaussianSplatRendererGroup() { OnDisable(); }

  bool OnEnable(const GsAssetDesc &asset, const std::vector<int> &cudaDevices, uint32_t flags = 0) {
    OnDisable();
    if (!ok(gs_group_create(cudaDevices.data(), (uint32_t)cudaDevices.size(), flags, &m_Group))) return false;
    m_Assets.assign(gs_group_local_count(m_Group), nullptr);
    if (!ok(gs_group_asset_upload(m_Group, &asset, m_Assets.data()))) return false;
    m_FrameCounter = 0;
    return true;
  }
  void OnDisable() {
    // the library owns the contexts: every object's assets go first
    for (GaussianSplatGroupObject *o : m_Objects) { for (GsAsset *a : o->m_Assets) if (a) gs_asset_destroy(a); delete o; }
    m_Objects.clear();
    for (GsAsset *a : m_Assets) if (a) gs_asset_destroy(a);
    m_Assets.clear();
    if (m_Group) gs_group_destroy(m_Group);
    m_Group = nullptr;
  }
  // Another splat object on the group (its asset uploaded to every member); owned by the group, nullptr on failure.
  GaussianSplatGroupObject *AddObject(const GsAssetDesc &asset) {
    GaussianSplatGroupObject *o = new GaussianSplatGroupObject();
    o->m_Assets.assign(gs_group_local_count(m_Group), nullptr);
    if (!m_Group || !ok(gs_group_asset_upload(m_Group, &asset, o->m_Assets.data()))) { delete o; return nullptr; }
    m_Objects.push_back(o);
    return o;
  }
  // Another splat object drawing the asset of `source` (this group or one of its objects): on every member an instance of
  // source's asset (gs_asset_instance), sharing its blobs in HBM.  Owned by the group, nullptr on failure.
  GaussianSplatGroupObject *AddInstance(const GaussianSplatGroupObject &source) {
    if (!m_Group || source.m_Assets.size() != m_Assets.size()) return nullptr;
    GaussianSplatGroupObject *o = new GaussianSplatGroupObject();
    o->m_Assets.assign(m_Assets.size(), nullptr);
    for (size_t i = 0; i < m_Assets.size(); ++i) {
      if (!ok(gs_asset_instance(source.m_Assets[i], &o->m_Assets[i]))) {
        for (GsAsset *a : o->m_Assets) if (a) gs_asset_destroy(a);
        delete o;
        return nullptr;
      }
    }
    m_Objects.push_back(o);
    return o;
  }
  // rts[i]: the image of local member i (device, host or CUDA-array memory) or nullptr
  bool SortAndRenderSplats(const CameraState &cam, GsImage *const *rts) {
    const int doSort = nextDoSort();
    GsFrameParams fp = params(cam);
    return ok(gs_group_frame(m_Group, m_Assets.data(), &fp, &options, doSort, rts));
  }
  // OnPreCullCamera on the group (R/GaussianSplatRenderer.cs:187-211): `objects` (this group and / or AddObject's) drawn in
  // GatherSplatsForCamera order (:73-105) into one target, then composited onto cameraTargets[i] (may be nullptr / hold nullptrs).
  bool SortAndRenderSplatsMulti(const CameraState &cam, std::vector<GaussianSplatGroupObject *> objects, GsImage *const *rts,
                                GsImage *const *cameraTargets = nullptr) {
    if (objects.empty()) return true;   // no active splat object: OnPreCullCamera draws nothing
    std::vector<GsAsset *> assets;
    std::vector<GsFrameParams> fps;
    std::vector<int32_t> doSort;
    if (!GatherObjects(cam, std::move(objects), assets, fps, doSort)) return false;
    return ok(gs_group_frame_objects(m_Group, (uint32_t)fps.size(), assets.data(), fps.data(), doSort.data(), &options, rts, cameraTargets));
  }
  // The render-thread event of SortAndRenderSplatsMulti: fills *out with the payload of GS_UNITY_EVENT_GROUP_FRAME_OBJECTS
  // (status GS_ERR_NOT_READY) with the same checks, GatherSplatsForCamera order and frame-counter steps; rts / cameraTargets
  // (each may be nullptr or hold nullptrs) are copied by value, one image per local member.  Returns false, with no frame
  // counter moved, where SortAndRenderSplatsMulti would return false before drawing, or draw nothing (no object).
  bool FillFrameObjectsEvent(const CameraState &cam, std::vector<GaussianSplatGroupObject *> objects, GsImage *const *rts,
                             GsImage *const *cameraTargets, UnityGroupFrameObjectsEvent *out) {
    if (!out || objects.empty() || !GatherObjects(cam, std::move(objects), out->assets, out->fps, out->doSort)) return false;
    const size_t L = m_Assets.size();
    out->rts.assign(L, GsImage{});
    out->cameraTargets.assign(L, GsImage{});
    for (size_t i = 0; i < L; ++i) {
      if (rts && rts[i]) out->rts[i] = *rts[i];
      if (cameraTargets && cameraTargets[i]) out->cameraTargets[i] = *cameraTargets[i];
    }
    GsUnityGroupFrameObjectsEvent &ev = out->event;
    std::memset(&ev, 0, sizeof(ev));
    ev.group = m_Group;
    ev.object_count = (uint32_t)out->fps.size();
    ev.assets = out->assets.data();
    ev.fps = out->fps.data();
    ev.do_sort = out->doSort.data();
    ev.options = options;
    ev.rts = rts ? out->rts.data() : nullptr;
    ev.camera_targets = cameraTargets ? out->cameraTargets.data() : nullptr;
    ev.status = GS_ERR_NOT_READY;
    return true;
  }
  // The payload of GS_UNITY_EVENT_GROUP_SYNC (Sync on the render thread).
  GsUnityGroupSyncEvent SyncEvent() const {
    GsUnityGroupSyncEvent ev;
    std::memset(&ev, 0, sizeof(ev));
    ev.group = m_Group;
    ev.status = GS_ERR_NOT_READY;
    return ev;
  }
  bool Sync() { return ok(gs_group_sync(m_Group)); }
  GsGroup *group() const { return m_Group; }
  GsAsset *asset(size_t i) const { return m_Assets[i]; }

 private:
  // gs_group_frame_objects' per-object arguments: `objects` in GatherSplatsForCamera order (:73-105), frame counters advanced.
  // False, with none moved, for a null object or one uploaded to another number of members.
  bool GatherObjects(const CameraState &cam, std::vector<GaussianSplatGroupObject *> objects, std::vector<GsAsset *> &assets,
                     std::vector<GsFrameParams> &fps, std::vector<int32_t> &doSort) const {
    auto depth = [&](const GaussianSplatGroupObject *o) {   // camera-space z of the object's position, +z forward
      const float *v = cam.worldToCameraMatrix.m, *p = o->localToWorldMatrix.m + 12;
      return -(v[2] * p[0] + v[6] * p[1] + v[10] * p[2] + v[14]);
    };
    const size_t L = m_Assets.size();
    for (const GaussianSplatGroupObject *o : objects)   // checked before any object's frame counter moves
      if (!o || o->m_Assets.size() != L) return false;
    std::stable_sort(objects.begin(), objects.end(), [&](const GaussianSplatGroupObject *a, const GaussianSplatGroupObject *b) {
      if (a->m_RenderOrder != b->m_RenderOrder) return a->m_RenderOrder > b->m_RenderOrder;
      return depth(a) < depth(b);
    });
    assets.clear(); fps.clear(); doSort.clear();
    for (GaussianSplatGroupObject *o : objects) {
      assets.insert(assets.end(), o->m_Assets.begin(), o->m_Assets.end());
      fps.push_back(o->params(cam));
      doSort.push_back(o->nextDoSort());
    }
    return true;
  }
  bool ok(int rc) const {
    if (rc == GS_OK) return true;
    std::fprintf(stderr, "GaussianSplatRendererGroup: %s (%d)\n", gs_last_error(m_Group ? gs_group_context(m_Group, 0) : nullptr), rc);
    return false;
  }
  GsGroup *m_Group = nullptr;
  std::vector<GaussianSplatGroupObject *> m_Objects;
};

}  // namespace GaussianSplatting
