/* gsplat_b200.h -- C ABI of the H100-native Gaussian-splat render path.
 *
 * This is the drop-in boundary for the hot path of aras-p/UnityGaussianSplatting
 * (view-calc -> depth sort -> rasterise/blend -> composite).  The reference has no
 * native plugin (SURVEY.md section 0, F3): all GPU work is recorded by C# into a Unity
 * CommandBuffer.  Every entry point below therefore replaces a *C# call site* and
 * the compute/raster work it dispatches; the citation next to each symbol names it
 * (paths relative to the reference repo, R/ = package/Runtime, S/ = package/Shaders).
 *
 * Rules of the ABI:
 *   - plain C: pointers, sizes, PODs.  No C++/torch types.
 *   - every function returns a GsStatus (0 = ok, <0 = error) and never throws or
 *     aborts; gs_last_error() gives the text.  This mirrors the reference's
 *     "log and skip" behaviour (R/GaussianSplatRenderer.cs:361-369,447-448,655).
 *   - one GsContext per CUDA device; calls on one context are serialised by the caller.
 *     All work is enqueued on the context's stream; only gs_sync/gs_readback_* /
 *     host-memory images block.
 *   - matrices are float[16], column-major exactly like UnityEngine.Matrix4x4
 *     (element (row r, col c) at [c*4 + r]).
 */
#ifndef GSPLAT_B200_H
#define GSPLAT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define GS_API __declspec(dllexport)
#else
#define GS_API __attribute__((visibility("default")))
#endif

typedef struct GsContext GsContext;
typedef struct GsAsset GsAsset;

typedef enum GsStatus {
  GS_OK = 0,
  GS_ERR_INVALID_ARGUMENT = -1,
  GS_ERR_CUDA = -2,
  GS_ERR_OUT_OF_MEMORY = -3,
  GS_ERR_UNSUPPORTED_FORMAT = -4, /* a format enum outside R/GaussianSplatAsset.cs:31-81 */
  GS_ERR_NOT_READY = -5,          /* e.g. gs_render before gs_calc_view */
  GS_ERR_NO_DEVICE = -6
} GsStatus;

/* R/GaussianSplatAsset.cs:31-37 (VectorFormat), S/GaussianSplatting.hlsl:319-323 */
typedef enum GsVectorFormat { GS_VEC_FLOAT32 = 0, GS_VEC_NORM16 = 1, GS_VEC_NORM11 = 2, GS_VEC_NORM6 = 3 } GsVectorFormat;
/* R/GaussianSplatAsset.cs:51-57 (ColorFormat) */
typedef enum GsColorFormat { GS_COL_FLOAT32X4 = 0, GS_COL_FLOAT16X4 = 1, GS_COL_NORM8X4 = 2, GS_COL_BC7 = 3 } GsColorFormat;
/* R/GaussianSplatAsset.cs:70-81 (SHFormat); values >= 4 are clustered palettes */
typedef enum GsSHFormat { GS_SH_FLOAT32 = 0, GS_SH_FLOAT16 = 1, GS_SH_NORM11 = 2, GS_SH_NORM6 = 3, GS_SH_CLUSTER64K = 4,
                          GS_SH_CLUSTER32K = 5, GS_SH_CLUSTER16K = 6, GS_SH_CLUSTER8K = 7, GS_SH_CLUSTER4K = 8 } GsSHFormat;

/* The asset blobs exactly as GaussianSplatAsset exposes them
 * (R/GaussianSplatAsset.cs:219-237; uploaded by CreateResourcesForAsset,
 * R/GaussianSplatRenderer.cs:373-421).  Pointers are HOST memory, borrowed for the
 * duration of gs_asset_upload; the library copies everything to HBM.
 * `color` is the 2048-wide, 16x16-Morton-swizzled texture image
 * (R/GaussianSplatAsset.cs:152-160, S/GaussianSplatting.hlsl:181-194), row-major.
 * `chunks` may be NULL / chunk_bytes 0 (fully-float32 assets,
 * R/GaussianSplatRenderer.cs:391-405). */
typedef struct GsAssetDesc {
  uint32_t splat_count;
  uint32_t pos_format, scale_format, sh_format, color_format;
  const void *pos, *other, *sh, *color, *chunks;
  uint64_t pos_bytes, other_bytes, sh_bytes, color_bytes, chunk_bytes;
} GsAssetDesc;

/* R/GaussianCutout.cs:20-40, S/SplatUtilities.compute:96-100 (68 bytes) */
typedef struct GsCutout {
  float mat[16];            /* cutout worldToLocal * renderer localToWorld */
  uint32_t type_and_flags;  /* low byte: 0 ellipsoid, 1 box, 0xFF ignore; 0x100: invert */
} GsCutout;

/* Per-frame uniforms.  Field-by-field these are the values C# binds in
 * CalcViewData (R/GaussianSplatRenderer.cs:579-610), SortPoints (:612-639) and
 * SortAndRenderSplats (:137-149). */
typedef struct GsFrameParams {
  float mat_object_to_world[16];  /* tr.localToWorldMatrix            (:587) */
  float mat_world_to_object[16];  /* tr.worldToLocalMatrix            (:588) */
  float mat_view[16];             /* cam.worldToCameraMatrix, -z fwd  (:586,:617) */
  float mat_proj_gpu[16];         /* UNITY_MATRIX_P = GL.GetGPUProjectionMatrix(cam.projectionMatrix, true);
                                     an engine global in the reference (S/SplatUtilities.compute:200,236) */
  float screen_w, screen_h;       /* _VecScreenParams.xy              (:591).  In [1, 16384] per axis, the largest
                                     render texture D3D12 makes (a splat's bin rectangle holds 8-bit indices of 64-pixel bins);
                                     anything else is GS_ERR_INVALID_ARGUMENT.  A screen above 8160 px (128 bins) on either
                                     axis makes the draw wait for the device once after binning: see "Bin-list capacity"
                                     below. */
  float cam_pos_world[3];         /* _VecWorldSpaceCameraPos          (:592) */
  float splat_scale;              /* m_SplatScale   [0.1,2]           (:599) */
  float opacity_scale;            /* m_OpacityScale [0.05,20]         (:600) */
  uint32_t sh_order;              /* m_SHOrder 0..3                   (:601) */
  uint32_t sh_only;               /* m_SHOnly                         (:602) */
  uint32_t cutout_count;          /* _SplatCutoutsCount (R/GaussianSplatRenderer.cs:506-508) */
  uint32_t reserved0;
  const GsCutout *cutouts;        /* host pointer, cutout_count entries, may be NULL */
  const uint32_t *deleted_bits;   /* host pointer, ceil(N/32) words or NULL == _SplatBitsValid 0 (:496-501) */
  const uint32_t *selected_bits;  /* host pointer, ceil(N/32) words or NULL: the edit selection (_SplatSelectedBits, :496).  A
                                     selected splat is drawn by the pixel shader's "selected" branch: magenta outline + tint,
                                     opacity from the gaussian alone (S/RenderGaussianSplats.shader:63-73,87-101) */
  const float *scene_depth;       /* optional: the camera's depth buffer the splat pass tests against.  The reference binds the
                                     current depth target beside _GaussianSplatRT (R/GaussianSplatRenderer.cs:195) and keeps
                                     ShaderLab's default ZTest LEqual with ZWrite Off (S/RenderGaussianSplats.shader:8-12), so
                                     splats behind opaque scene geometry are not drawn.  screen_w x screen_h float32, rows
                                     tightly packed, in mat_proj_gpu's convention (reversed Z: 1 = near plane), where LEqual is
                                     evaluated as "fragment depth >= stored depth"; every fragment of a splat has the depth
                                     clip.z / clip.w of its centre (the quad is flat).  NULL = no depth test. */
  uint32_t scene_depth_on_device; /* the GsMemory of scene_depth.  0 (GS_MEM_HOST): host memory, uploaded per frame.
                                     GS_MEM_ARRAY (2): scene_depth is a cudaArray_t, a 2-D array of screen_w x screen_h (depth 0)
                                     of one 32-bit float channel, created with cudaArraySurfaceLoadStore.  GS_MEM_ARRAY_LAYER (4):
                                     scene_depth points to a borrowed GsArrayLayer naming one layer of a layered array of
                                     screen_w x screen_h of one 32-bit float channel, created with cudaArrayLayered |
                                     cudaArraySurfaceLoadStore (`layer` below its layer count, `reserved` 0) -- e.g. one eye of an XR
                                     eye-depth array.  Texel (x, y) of the array (layer) is the depth of pixel (x, y), read in place.
                                     Another channel format is GS_ERR_UNSUPPORTED_FORMAT; any other mismatch, a null array, or a
                                     layered array passed as 2 (a 2-D one as 4) is GS_ERR_INVALID_ARGUMENT, refused before anything
                                     is enqueued.  GS_MEM_ARRAY_RECT (5): scene_depth points to a borrowed GsArrayRect over a
                                     2-D or layered array of one 32-bit float channel made with cudaArraySurfaceLoadStore; the
                                     rectangle is screen_w x screen_h at (x, y) and must lie inside the array, and texel
                                     (x + px, y + py) of the layer is the depth of pixel (px, py) -- e.g. the camera's depth in
                                     an HDRP RTHandle allocated larger than the camera.  The group entry points (gs_group_*)
                                     refuse 2, 4 and 5 (GS_ERR_INVALID_ARGUMENT).
                                     Any other value (1, 3, 6, ...): device memory, used in place. */
  uint32_t reserved1;
} GsFrameParams;

/* GS_PIX_B10G11R11_UFLOAT: one 32-bit texel per pixel, no alpha: R in bits 0-10 and G in bits 11-21 (unsigned float11), B in
 * bits 22-31 (unsigned float10) -- Unity's B10G11R11_UFloatPack32, VK_FORMAT_B10G11R11_UFLOAT_PACK32,
 * DXGI_FORMAT_R11G11B10_FLOAT: the HDR colour buffer of URP and HDRP cameras.  It is accepted as a CAMERA TARGET, in every
 * memory kind: gs_composite's camera_target, the camera targets of gs_frame, gs_frame_objects and gs_frame_cameras,
 * gs_group_frame_objects' camera_targets (and so the camera_target of GsUnityFrameEvent / GsUnityFrameObjectsEvent).  A CUDA
 * array holding it has ONE 32-bit cudaChannelFormatKindUnsigned channel (cudaCreateChannelDesc<unsigned int>()); any other
 * channel format is GS_ERR_UNSUPPORTED_FORMAT, as a uint32 array is for an RGBA16F / RGBA32F image.  It is refused with
 * GS_ERR_UNSUPPORTED_FORMAT, before anything is enqueued, as any render target (rt, rts[], a group's rts), as gs_composite's
 * rt, as band_packed output and as gs_unshuffle_bands' out.
 * The composite onto it decodes the texel, blends r, g and b exactly as onto an RGBA16F / RGBA32F target, drops alpha and
 * encodes; a pixel whose source alpha is not > 0 keeps its bits.  Each channel has 5 exponent bits (bias 15) and 6 (float11)
 * or 5 (float10) mantissa bits:
 *   decode  exact: exponent 0 is mantissa * 2^-14 / 2^m (denormals), exponent 31 is +Inf with mantissa 0, else NaN;
 *   encode  NaN -> all ones (0x7FF / 0x3FF); any value <= 0, -0 and -Inf included -> 0; +Inf -> 0x7C0 / 0x3E0; anything else
 *           rounds to nearest, ties to even, over the whole value set including denormals, and overflows to +Inf as IEEE
 *           rounding does: float11 x >= 65280 (largest finite 65024), float10 x >= 65024 (largest finite 64512).
 * This follows the format definitions of the Vulkan and D3D11 specifications, and rounds as the RGBA16F path's
 * float -> half conversion does; whether a given GPU's blend unit rounds this format the same way is not known here.
 *
 * GS_PIX_R8G8B8A8_SRGB: four bytes per pixel in memory order R, G, B, A; R, G and B sRGB-encoded, A linear UNorm -- Unity's
 * R8G8B8A8_SRGB, VK_FORMAT_R8G8B8A8_SRGB, DXGI_FORMAT_R8G8B8A8_UNORM_SRGB: the colour buffer of an LDR camera (HDR off) in a
 * linear-colour-space project, and the render texture the reference's GaussianSplatValidator renders into.  Like
 * GS_PIX_B10G11R11_UFLOAT it is accepted as a CAMERA TARGET only, in every memory kind, by the same entry points (and so by the
 * camera targets of every GsUnity*Event), and refused with GS_ERR_UNSUPPORTED_FORMAT, before anything is enqueued, wherever
 * GS_PIX_B10G11R11_UFLOAT is.  A CUDA array holding it has FOUR 8-bit cudaChannelFormatKindUnsigned channels
 * (cudaCreateChannelDesc<uchar4>()); any other channel format is GS_ERR_UNSUPPORTED_FORMAT.  A pitched linear image follows the
 * pitch rules with a 4-byte texel.
 * The composite onto it decodes the texel, blends r, g, b and a exactly as onto an RGBA32F target (alpha included:
 * o.a = fma(a, a, d.a * (1 - a))) and encodes; a pixel whose source alpha is not > 0 keeps its bytes.  The codec is exact:
 *   decode  RGB: code c -> the float32 nearest the IEC 61966-2-1 EOTF at v = c / 255, the exact value of v / 12.92 for
 *           v <= 0.04045, else ((v + 0.055) / 1.055)^2.4 (a 256-entry table);  A: code a -> the float32 nearest a / 255;
 *   encode  RGB: NaN and x <= 0 (-0 and -Inf included) -> 0; x >= 1 (+Inf included) -> 255; any other x -> the number of j in
 *           1..255 with 255 OETF(x) >= j - 0.5, evaluated exactly, where OETF(x) = 12.92 x for x <= 0.0031308, else
 *           1.055 x^(1/2.4) - 0.055: round to nearest in the encoded domain.  Equivalently x is compared with 255 float32
 *           thresholds T_j, the smallest float32 with 255 OETF(T_j) >= j - 0.5.  The OETF falls by 2.9e-8 at its junction, but
 *           no decision boundary lies in that step, so the code is monotone in x;
 *           A: NaN -> 0; else clamp to [0, 1] and round 255 x to nearest (the only representable tie, x = 0.5, gives 128).
 * Whether a given GPU's blend unit rounds this format the same way is not known here: D3D and Vulkan allow some tolerance in
 * the sRGB conversion. */
typedef enum GsPixelFormat {
  GS_PIX_RGBA16F = 0,   /* _GaussianSplatRT: R16G16B16A16_SFloat (R/GaussianSplatRenderer.cs:194) */
  GS_PIX_RGBA32F = 1,
  GS_PIX_B10G11R11_UFLOAT = 2,   /* camera targets only (above) */
  GS_PIX_R8G8B8A8_SRGB = 3       /* camera targets only (above) */
} GsPixelFormat;

/* GS_MEM_ARRAY (images only, not GsPackDesc / GsPackedAsset): `data` is a cudaArray_t -- a 2-D CUDA array (mip level 0) on the
 * context's device, e.g. a Vulkan / D3D12 render texture imported with cudaImportExternalMemory +
 * cudaExternalMemoryGetMappedMipmappedArray + cudaGetMipmappedArrayLevel(.., 0), or a GL / D3D11 one from
 * cudaGraphicsSubResourceGetMappedArray.  The library reads and writes it in place through surface objects, so:
 *   - the array must have been created with cudaArraySurfaceLoadStore (for an imported image: ask for that flag in
 *     cudaExternalMemoryMipmappedArrayDesc.flags);
 *   - its channel format must be the image's: 4 x 16-bit float for GS_PIX_RGBA16F, 4 x 32-bit float for GS_PIX_RGBA32F,
 *     1 x 32-bit unsigned for GS_PIX_B10G11R11_UFLOAT, 4 x 8-bit unsigned for GS_PIX_R8G8B8A8_SRGB
 *     (else GS_ERR_UNSUPPORTED_FORMAT);
 *   - its extent must be width x height with depth 0, and row_pitch_bytes must be 0 (else GS_ERR_INVALID_ARGUMENT).
 * The import itself and the graphics API's semaphores stay with the host: wait / signal them on gs_context_stream(ctx).
 * Not accepted (GS_ERR_INVALID_ARGUMENT): band_packed output and gs_unshuffle_bands output.  GS_FLAG_ASYNC_READBACK has no
 * effect on an array render target (it applies to host images only). */
typedef enum GsMemory { GS_MEM_HOST = 0, GS_MEM_DEVICE = 1, GS_MEM_ARRAY = 2 } GsMemory;

/* GS_MEM_ARRAY_LAYER (images only): `data` points to a GsArrayLayer, a host descriptor borrowed for the call, that names one
 * layer of a layered CUDA array -- e.g. one eye of an XR eye-texture array in single-pass-instanced mode, or one face of a
 * cube map, imported with extent.depth = its layer count and flags cudaArrayLayered | cudaArraySurfaceLoadStore.  The layer is
 * rendered into / composited onto in place through a layered surface; the array's other layers are not touched.  The rules of
 * GS_MEM_ARRAY apply, except that:
 *   - the array must have been created with cudaArrayLayered | cudaArraySurfaceLoadStore, with extent width x height, and
 *     `layer` must be below its depth (its layer count); `reserved` must be 0 (else GS_ERR_INVALID_ARGUMENT).
 * A layered array passed as GS_MEM_ARRAY is GS_ERR_INVALID_ARGUMENT, as is a 2-D array passed as GS_MEM_ARRAY_LAYER.
 * Memory kind 3 is not defined (GS_ERR_INVALID_ARGUMENT). */
#define GS_MEM_ARRAY_LAYER 4u
typedef struct GsArrayLayer {
  void *array;      /* a layered cudaArray_t (mip level 0) on the context's device */
  uint32_t layer;   /* the layer drawn into, below the array's layer count */
  uint32_t reserved;
} GsArrayLayer;

/* GS_MEM_ARRAY_RECT (images only): `data` points to a GsArrayRect, a host descriptor borrowed for the call, that names a
 * width x height rectangle of a 2-D CUDA array or of one layer of a layered one.  Pixel (px, py) of the image is texel
 * (x + px, y + py) of the layer; the texels outside the rectangle, and the other layers, are not touched.  Two uses:
 *   - a render target larger than the camera: HDRP allocates its RTHandles at the largest size any camera has needed, and each
 *     camera draws into the rectangle at the texture's origin, at its (dynamically scaled) pixel size: GsArrayRect{array, 0, 0, 0,
 *     0} with that size as the image's width x height and as screen_w x screen_h;
 *   - several views in one texture (split screen, impostor or probe atlases, the quilt of a light-field display): one
 *     rectangle per camera of gs_frame_cameras, which draws disjoint rectangles of one array in one camera run.
 * Whether the array is 2-D or layered is read from it (cudaArrayGetInfo).  The rules of GS_MEM_ARRAY apply (channel format,
 * cudaArraySurfaceLoadStore, row_pitch_bytes 0, not accepted as band_packed or gs_unshuffle_bands output), except for the
 * extent: the rectangle must lie inside the array.  GS_ERR_INVALID_ARGUMENT, before anything is enqueued: a null array,
 * `reserved` not 0, a nonzero `layer` of a 2-D array, a layer not below a layered array's layer count, a 3-D array that is not
 * layered, a rectangle that does not lie inside the array.  A camera's rt and camera target must not overlap (the library
 * does not check this, as for whole arrays).  Memory kinds 3 and above 5 are not defined (GS_ERR_INVALID_ARGUMENT). */
#define GS_MEM_ARRAY_RECT 5u
typedef struct GsArrayRect {
  void *array;       /* a 2-D or layered cudaArray_t (mip level 0) on the context's device */
  uint32_t layer;    /* 0 for a 2-D array; below the layer count of a layered one */
  uint32_t x, y;     /* texel of the array that holds pixel (0, 0) of the image */
  uint32_t reserved; /* 0 */
} GsArrayRect;       /* 24 bytes */

typedef struct GsImage {
  void *data;                /* host pointer, device pointer, cudaArray_t (GS_MEM_ARRAY), GsArrayLayer * (GS_MEM_ARRAY_LAYER) or
                                GsArrayRect * (GS_MEM_ARRAY_RECT) */
  uint32_t width, height;
  uint32_t row_pitch_bytes;  /* 0 = tightly packed (and always 0 for the CUDA-array kinds 2, 4 and 5) */
  uint32_t format;           /* GsPixelFormat */
  uint32_t memory;           /* GsMemory, GS_MEM_ARRAY_LAYER or GS_MEM_ARRAY_RECT: where `data` lives; any other value is
                                GS_ERR_INVALID_ARGUMENT */
} GsImage;

/* How the render-target blend is evaluated.
 * GS_BLEND_FP16_ROP reproduces the reference: the RT is RGBA16F, so the fixed-function
 * blender (Blend OneMinusDstAlpha One, S/RenderGaussianSplats.shader:11) rounds dst to
 * half after EVERY splat.  GS_BLEND_FP32 keeps dst in float32 registers and rounds once. */
typedef enum GsBlendMode { GS_BLEND_FP16_ROP = 0, GS_BLEND_FP32 = 1 } GsBlendMode;

#define GS_BAND_PIXELS 64u /* height of one partition row = edge of a binning cell (csrc/gs_common.cuh kBin) */
#define GS_TILE_PIXELS 16u /* edge of a raster tile = granularity of row_begin/row_end (csrc/gs_common.cuh kTile) */

typedef struct GsRenderOptions {
  uint32_t blend_mode;        /* GsBlendMode */
  uint32_t band_packed;       /* 1: rt holds only this partition's rows, packed: own 64-pixel row k -> pixel rows
                                 [64k, 64k+64); rt->height must be 64 * (number of own rows).  This is the
                                 send buffer of the all-gather. */
  /* Screen-tile partition for multi-GPU (SURVEY 8e.1): this context composites only
   * 64-pixel rows (GS_BAND_PIXELS, the binning cell) r with (r / band_rows) % partition_count == partition_index.
   * partition_count 0 or 1 = whole image. */
  uint32_t partition_index, partition_count, band_rows;
  uint32_t flags;             /* GsRenderFlags */
  /* Contiguous partition (what gs_group_frame uses): when row_end > row_begin this context composites only the 16-pixel
   * raster-tile rows [row_begin, row_end) (GS_TILE_PIXELS), straight into their natural place of a full-size target;
   * partition_* and band_packed are then ignored.  0,0 = not used. */
  uint32_t row_begin, row_end;
} GsRenderOptions;

typedef enum GsRenderFlags {
  /* gs_frame with a HOST render target (the flag has no effect on device or array targets) returns as soon as the read-back is ENQUEUED (on a second stream, double-buffered
   * device staging): frame k's copy overlaps frame k+1's kernels.  The image must be pinned (cudaHostRegister /
   * cudaMallocHost) and must not be read, nor handed to another frame, until gs_sync (or two later frames) -- the
   * managed-side analogue is AsyncGPUReadback.  Errors of the frame (e.g. a truncated bin list) surface at gs_sync. */
  GS_FLAG_ASYNC_READBACK = 1u,
  /* Do not start from a cleared target: read `rt` and blend this asset UNDER what is already there.  The reference
   * clears _GaussianSplatRT once per camera (R/GaussianSplatRenderer.cs:196) and then draws every active splat object
   * into it, nearest object first (GatherSplatsForCamera :73-105, loop :111-168): render the first object without this
   * flag and each further one with it.  A host `rt` is uploaded first. */
  GS_FLAG_LOAD_RT = 2u
} GsRenderFlags;

/* Per-stage device times of the last gs_frame/gs_sort/gs_calc_view/gs_render call with
 * timing enabled (GaussianSplat.Sort / CalcView / Draw / Compose profiler markers,
 * R/GaussianSplatRenderer.cs:20-22,287).  Milliseconds, CUDA events on the context stream. */
typedef struct GsStageTimes {
  float distances_ms, sort_ms, view_ms, bin_ms, raster_ms, composite_ms, total_ms;
  float sort_pass_ms[4];
  uint64_t tile_entries;      /* (tile, splat) pairs produced by binning */
  uint32_t kernel_launches;   /* kernels of this library launched by the call */
  uint32_t reserved;
} GsStageTimes;

/* ---- lifetime ---------------------------------------------------------------- */
/* EnsureSorterAndRegister + resource setup, R/GaussianSplatRenderer.cs:450-475.
 * stream_handle: an existing cudaStream_t to enqueue on (0 = create a private stream). */
GS_API int gs_create(int cuda_device, void *stream_handle, GsContext **out);
GS_API void gs_destroy(GsContext *ctx);
GS_API const char *gs_last_error(GsContext *ctx); /* ctx may be NULL: last global error */
GS_API int gs_sync(GsContext *ctx);
GS_API int gs_set_timing(GsContext *ctx, int enabled);
GS_API int gs_get_stage_times(GsContext *ctx, GsStageTimes *out);
GS_API const char *gs_version(void);

/* ---- asset --------------------------------------------------------------------- */
/* CreateResourcesForAsset + InitSortBuffers + CSSetIndices,
 * R/GaussianSplatRenderer.cs:373-445, S/SplatUtilities.compute:59-67 */
GS_API int gs_asset_upload(GsContext *ctx, const GsAssetDesc *desc, GsAsset **out);
/* A further renderer of an uploaded asset: CreateResourcesForAsset (R/GaussianSplatRenderer.cs:373-445) for a
 * GaussianSplatRenderer whose m_Asset another renderer already has on this context.  *out behaves in every call exactly like an
 * asset gs_asset_upload made on source's context from the same GsAssetDesc, and starts as a fresh upload does: draw order
 * reset (CSSetIndices), no view data.  It shares source's five blobs in HBM (nothing is copied or allocated for them) and owns
 * its own per-renderer state: draw order, keys, view data, bin rectangles, draw records, quad depths and group buffers.
 * source may itself be an instance; the blobs are freed when the last asset holding them is destroyed, in any order.  A source
 * and its instances are distinct assets: one call may list several of them, and an instance of a group member's asset is that
 * member's asset in gs_group_frame / gs_group_frame_objects.  GS_ERR_INVALID_ARGUMENT for a NULL source or out;
 * GS_ERR_OUT_OF_MEMORY with *out NULL when the per-renderer buffers cannot be allocated.  Blocks. */
GS_API int gs_asset_instance(const GsAsset *source, GsAsset **out);
/* DisposeResourcesForAsset / OnDisable, R/GaussianSplatRenderer.cs:533-577.  An asset shared with instances keeps its blobs
 * alive for them. */
GS_API void gs_asset_destroy(GsAsset *asset);
/* CSSetIndices: order[i] = i (S/SplatUtilities.compute:59-67) */
GS_API int gs_asset_reset_order(GsAsset *asset);
GS_API uint32_t gs_asset_splat_count(const GsAsset *asset);

/* ---- the hot path -------------------------------------------------------------- */
/* SortPoints: CSCalcDistances + GpuSorting.Dispatch
 * (R/GaussianSplatRenderer.cs:612-639, S/SplatUtilities.compute:69-82,
 *  R/GpuSorting.cs:142-198).  The order buffer persists across calls: distances are
 * gathered through the previous order and the sort is stable, exactly as the reference. */
GS_API int gs_sort(GsContext *ctx, GsAsset *asset, const GsFrameParams *fp);
/* CalcViewData: CSCalcViewData (R/GaussianSplatRenderer.cs:579-610,
 * S/SplatUtilities.compute:189-252) */
GS_API int gs_calc_view(GsContext *ctx, GsAsset *asset, const GsFrameParams *fp);
/* cmb.DrawProcedural(matSplats, 6 idx, N instances) into the cleared _GaussianSplatRT
 * (R/GaussianSplatRenderer.cs:156-165,194-196; S/RenderGaussianSplats.shader).
 * Output: premultiplied RGBA (format/memory per `rt`).  Requires gs_calc_view first. */
GS_API int gs_render(GsContext *ctx, GsAsset *asset, const GsFrameParams *fp,
                     const GsRenderOptions *opt, GsImage *rt);
/* Composite pass: GaussianComposite.shader:35-39 with Blend SrcAlpha OneMinusSrcAlpha
 * (R/GaussianSplatRenderer.cs:206-210).  `camera_target` is read-modify-write. */
GS_API int gs_composite(GsContext *ctx, const GsImage *rt, GsImage *camera_target);
/* Bin-list capacity.  The draw lists one (bin, splat) entry per 64-pixel bin a splat's footprint touches, in a list of
 * clamp(8 x splats, 4 Mi, 768 Mi) entries (for gs_frame_objects, 8 x a run's summed splats).  A list that needs more is
 * truncated and the frame reports GS_ERR_OUT_OF_MEMORY: when the call reads its image back to the host, or else at gs_sync.
 * Screens above 8160 px (128 bins) on either axis are the exception: the rule was set for smaller screens, and a splat's
 * footprint in bins grows with the square of the screen size, so after binning the host waits for the device and reads the
 * entry count back: one wait per draw, per run of gs_frame_objects and per object of a group member's draw, which smaller
 * screens do not have (their calls return once the work is enqueued).  A list that overflowed is grown to the entries it needs plus a quarter, at most 768 Mi, and the frame is
 * binned again; the capacity is kept, so the next frames of that size bin once.  Beyond 768 Mi the frame reports GS_ERR_OUT_OF_MEMORY as above.
 * GsStageTimes.tile_entries is the count of the list the draw used. */

/* SortAndRenderSplats for one renderer, one stream, no host round trips:
 * (do_sort ? gs_sort : nothing) -> gs_calc_view -> gs_render [-> gs_composite if
 * camera_target != NULL].  do_sort == (m_FrameCounter % m_SortNthFrame == 0),
 * R/GaussianSplatRenderer.cs:120-121.  rt may be NULL when camera_target is given
 * (the RT then lives only in library scratch).
 * In the reference _SplatViewData only carries CSCalcViewData's results to the draw call; the fused
 * path hands them to its compositor directly and does NOT materialise that buffer (nor the colour of
 * splats that cannot produce a fragment).  Pixels are unaffected; gs_readback_view after gs_frame
 * returns GS_ERR_NOT_READY -- call gs_calc_view when the buffer itself is wanted. */
GS_API int gs_frame(GsContext *ctx, GsAsset *asset, const GsFrameParams *fp,
                    const GsRenderOptions *opt, int do_sort, GsImage *rt, GsImage *camera_target);
/* GaussianSplatRenderSystem.SortAndRenderSplats for one camera on one context (R/GaussianSplatRenderer.cs:73-105,108-169,
 * 187-211): the render target cleared once, every object drawn into it in the caller's order (GatherSplatsForCamera), then
 * one composite onto the camera target.
 *   Result: rt, camera_target and every object's persistent draw order are bit-identical to gs_frame(assets[0], flags 0),
 *   then gs_frame(assets[k], GS_FLAG_LOAD_RT) for k >= 1, then gs_composite(rt, camera_target) when camera_target is given --
 *   for both blend modes and both pixel formats.
 *   assets, fps, do_sort  [object_count]: each object's asset (of this context, each listed once), uniforms and
 *                   m_FrameCounter % m_SortNthFrame == 0.  All objects must share screen_w / screen_h.
 *   opt             blend_mode and GS_FLAG_ASYNC_READBACK (as gs_frame); may be NULL.
 *   rt, camera_target  host, device or CUDA-array memory, screen-sized; at least one must be given.
 * Per object, in order, on the context stream: the sort (when do_sort[k]) and the view-calc, as gs_frame.  Then consecutive
 * objects are drawn together as one run: their bin-list entries go into one list, object after object, which is sorted once
 * by bin id and drawn by one raster pass.  A run holds at most 16 objects, each with fewer than 2^28 splats, binding at most
 * one scene depth buffer (the same scene_depth pointer and memory; for CUDA arrays the same array, layer and rectangle); a new run starts where one of these would break, and
 * blends under what the earlier runs drew.  Any object count is accepted.  A run of one object (with one object: the whole
 * call) does the device work of gs_frame.  The bin-list capacity of a run is clamp(8 x its summed splat count, 4 Mi, 768 Mi)
 * entries; a run that needs more reports GS_ERR_OUT_OF_MEMORY as gs_frame does (at gs_sync when nothing is read back to the
 * host), even when a later run's list fits, except on screens above 8160 px, where the list grows first (see "Bin-list
 * capacity").
 * GsStageTimes after this call: bin_ms, raster_ms, composite_ms and tile_entries are those of the call's draw when it forms one
 * run; with several runs, bin_ms runs from the end of the last view-calc to the end of the last run's bin sort, and raster_ms
 * and tile_entries are the last run's.  distances_ms, sort_ms, sort_pass_ms and view_ms are those of the last object that
 * was sorted / view-calculated; total_ms spans the whole call; kernel_launches counts every kernel.
 * GS_ERR_INVALID_ARGUMENT, with nothing enqueued and nothing written: a NULL ctx, assets, fps or do_sort; object_count 0;
 * a NULL asset; an asset listed twice or of another context; objects of different screen sizes; GS_FLAG_LOAD_RT, a
 * partition, row_begin / row_end or band_packed in opt.  Image errors are reported as gs_frame reports them. */
GS_API int gs_frame_objects(GsContext *ctx, uint32_t object_count, GsAsset *const *assets, const GsFrameParams *fps,
                            const int32_t *do_sort, const GsRenderOptions *opt, GsImage *rt, GsImage *camera_target);
/* The camera loop of GaussianSplatRenderSystem (R/GaussianSplatRenderer.cs:187-211): OnPreCullCamera runs for every camera
 * but CameraType.Preview (:75, :581, :614) -- an editor's Scene and Game views, secondary views, one camera per eye (:590-591)
 * -- and each camera gathers and draws its own objects (GatherSplatsForCamera :73-105, SortAndRenderSplats :108-169).
 *   Result: bit-identical to
 *     for c: gs_frame_objects(ctx, object_counts[c], assets + off_c, fps + off_c, do_sort + off_c, opt, rts[c], camera_targets[c])
 *   with off_c = object_counts[0] + ... + object_counts[c - 1]: every render target, every camera target, and every asset's
 *   persistent draw order and sorted keys, for both blend modes and both pixel formats.  An asset's draw order is one buffer
 *   shared by every camera (m_GpuSortKeys, :142) and m_FrameCounter advances once per camera (:120-122), so a camera's sort
 *   gathers its distances through the order the previous camera's sort left, and the stable sort breaks ties by it; with
 *   m_SortNthFrame > 1 a camera that does not sort draws in the previous camera's order.  Both hold here.
 *   object_counts [camera_count]: the objects of each camera, at least one.
 *   assets, fps, do_sort: camera-major; camera c's objects, in its GatherSplatsForCamera order, are entries
 *                   [off_c, off_c + object_counts[c]).  Each camera's objects share that camera's screen size; cameras may
 *                   have different sizes.  An asset may appear in several cameras but only once within one.
 *   opt             blend_mode (as gs_frame_objects); may be NULL.
 *   rts, camera_targets [camera_count]: the cameras' images (host, device or CUDA-array memory, screen-sized); either of a
 *                   camera's two may be NULL, not both.
 * Consecutive cameras are drawn together as a camera run: per camera and per object in order, on the context stream, the
 * sort (when do_sort), the view-calc and that object's bin-list entries (bin ids offset by the camera's first bin in the run);
 * then one stable sort of the run's list by bin id, one raster pass over the tiles of all its cameras (the longest tiles of
 * all cameras first), and per camera the host read-back and the composite.  The records of an asset that a later camera of
 * the run draws again are kept in a context scratch slab until the raster.  A run holds at most 16 (camera, object) pairs,
 * each object under 2^28 splats, cameras of at most 8160 px per axis and 65536 64-pixel bins in all, at most one scene depth
 * buffer per camera, and one render-target pixel format (RGBA16F for a camera without rt).  A camera whose rt or camera
 * target is the render target of an earlier camera of the run starts a new run; for CUDA arrays "is" means the same array
 * and layer with overlapping rectangles (a whole array or layer overlaps every rectangle of it), so cameras drawing into
 * disjoint GS_MEM_ARRAY_RECT tiles of one array share a run.  A camera that breaks a limit of its own (a
 * larger screen, more objects or splats, two depth buffers), and a camera that ends up alone in its run, is drawn by
 * gs_frame_objects' own work, large screens' bin-list growth included.  A run's bin-list capacity is
 * clamp(8 x its summed splats over all pairs, 4 Mi, 768 Mi) entries; overflow is reported as gs_frame_objects reports it
 * (when the call reads a host image back, else at gs_sync), for any run of the call.
 * GsStageTimes after this call follows gs_frame_objects' rules for several runs: bin_ms runs from the end of the last
 * view-calc to the end of the last run's bin sort (in a camera run each object's entries are emitted right after its
 * view-calc, so this holds the last object's emit and the run's sort), raster_ms and tile_entries are the last run's,
 * composite_ms runs from the end of the last raster to the end of the last composite, total_ms (like gs_frame_objects') from
 * the start of the last sort or view-calc to the end of the call, and kernel_launches counts every kernel.  With one camera
 * the call does gs_frame_objects' device work, kernel for kernel.
 * GS_ERR_INVALID_ARGUMENT, with nothing enqueued and nothing written: everything gs_frame_objects refuses, for any camera; a
 * NULL object_counts, rts or camera_targets array; camera_count 0; a camera without objects; GS_FLAG_ASYNC_READBACK
 * (per-camera double-buffered staging is not provided: host images are read back before the call returns). */
GS_API int gs_frame_cameras(GsContext *ctx, uint32_t camera_count, const uint32_t *object_counts, GsAsset *const *assets,
                            const GsFrameParams *fps, const int32_t *do_sort, const GsRenderOptions *opt, GsImage *const *rts,
                            GsImage *const *camera_targets);

/* Multi-GPU epilogue (SURVEY 8e.1): `gathered` is the all-gather of every partition's band-packed
 * render target, [partition_count][rows_per_partition][width] pixels in DEVICE memory, where
 * rows_per_partition = 64 * max over partitions of own 64-pixel rows.  Writes the assembled width x height
 * image (device or host) in normal row order. */
GS_API int gs_unshuffle_bands(GsContext *ctx, const void *gathered, uint32_t partition_count, uint32_t band_rows,
                              uint32_t rows_per_partition, uint32_t pixel_format, GsImage *out);

/* ---- several GPUs of one box (SURVEY 8e; the reference itself is single-GPU) ----------------------------------
 * A group renders ONE frame on G GPUs and leaves, on every GPU, exactly what gs_frame leaves on one: the same draw order
 * (bit for bit: the persistent _SplatSortKeys contract of R/GpuSorting.cs:142-198 seeded by last frame's order,
 * R/GaussianSplatRenderer.cs:612-639) and the same render target.  Per frame and GPU:
 *   - the depth sort is sharded by KEY RANGE: every GPU computes the (cheap) key table, takes the splats whose key lies
 *     between two shared splitters -- in last frame's order, so ties keep the reference's order -- sorts only those, and one
 *     exchange of the id slabs gives every GPU the whole order (SURVEY 8e.2).  After gs_group_join the slabs travel as
 *     peer-to-peer stores over NVLink into CUDA-IPC mappings of the peers' order buffers (no collective call); groups made
 *     by gs_group_create, and boxes without IPC, use one ncclAllGather;
 *   - view-calc, binning and compositing are sharded by SCREEN ROWS: a contiguous range of 16-pixel rows per GPU
 *     (GsRenderOptions.row_begin/row_end), rebalanced every frame from the measured per-row cost, composited straight
 *     into place, then one NCCL exchange of the row ranges (SURVEY 8e.1: "a single all-gather of the composited tile buffers";
 *     grouped broadcasts of the exact sizes, in place, on a transfer stream that overlaps the next frame's sort).
 * Two ways to form a group:
 *   gs_group_join    one process per GPU (torchrun-style): every process passes its own context, the group size, its rank
 *                    and the 128-byte id rank 0 got from gs_group_unique_id (sent over any host channel);
 *   gs_group_create  one process driving n GPUs (what a Unity host would do): the library creates the n contexts.
 *                    GS_GROUP_EMULATE lets device indices repeat: the "GPUs" are then n contexts on the same device and the
 *                    exchanges are device-to-device copies -- the whole sharded path on a single-GPU box, for tests.
 * NCCL is bound at run time (libnccl.so.2; a copy already loaded into the process, e.g. PyTorch's, is reused). */
typedef struct GsGroup GsGroup;
#define GS_GROUP_ID_BYTES 128u
#define GS_GROUP_MAX_GPUS 16u
typedef enum GsGroupFlags { GS_GROUP_EMULATE = 1u } GsGroupFlags;

typedef struct GsGroupStats {      /* of the first local member, last gs_group_frame with timing enabled (gs_set_timing) */
  float distances_ms, slab_sort_ms, order_exchange_ms, view_ms, bin_ms, raster_ms, image_exchange_ms, total_ms;
  uint32_t group_size, rank;
  uint32_t row_bounds[GS_GROUP_MAX_GPUS + 1];   /* 16-pixel row ranges of this frame: GPU g composites [row_bounds[g], row_bounds[g+1]) */
  uint32_t slab_counts[GS_GROUP_MAX_GPUS];      /* splats each GPU sorted this frame */
} GsGroupStats;

GS_API int gs_group_unique_id(void *id_out /* GS_GROUP_ID_BYTES */);
GS_API int gs_group_join(GsContext *ctx, uint32_t group_size, uint32_t rank, const void *id, GsGroup **out);
GS_API int gs_group_create(const int *cuda_devices, uint32_t n, uint32_t flags, GsGroup **out);
GS_API void gs_group_destroy(GsGroup *group);
GS_API uint32_t gs_group_size(const GsGroup *group);
GS_API uint32_t gs_group_local_count(const GsGroup *group);          /* members driven by this process: 1 after join, n after create */
GS_API GsContext *gs_group_context(GsGroup *group, uint32_t local_index);
/* CreateResourcesForAsset on every local member (R/GaussianSplatRenderer.cs:373-445): assets_out[local_count]. */
GS_API int gs_group_asset_upload(GsGroup *group, const GsAssetDesc *desc, GsAsset **assets_out);
/* SortAndRenderSplats (R/GaussianSplatRenderer.cs:108-169) on the group.  assets[i] / rts[i] belong to local member i;
 * rts[i] is a full-size image (device, host or CUDA-array memory; NULL = this member keeps the frame in library scratch only).
 * Every non-NULL rts[i] ends up holding the COMPLETE render target; an array is filled by one copy of the assembled frame on the
 * member's transfer stream, complete after gs_group_sync.  `opt`: blend_mode, and GS_FLAG_ASYNC_READBACK for host images
 * (the call returns with the read-back enqueued; gs_group_sync completes it).  Collective: every process of the
 * group must call it with the same parameters. */
GS_API int gs_group_frame(GsGroup *group, GsAsset *const *assets, const GsFrameParams *fp, const GsRenderOptions *opt, int do_sort,
                          GsImage *const *rts);
/* One camera's frame with several splat objects on the group: OnPreCullCamera (R/GaussianSplatRenderer.cs:187-211) -- the
 * render target cleared once, every active object sorted, view-calculated and drawn into it in the caller's order
 * (GatherSplatsForCamera, :73-105, loop :111-168), then the composite onto the camera target.  Every member ends with exactly
 * what one GPU leaves after gs_frame per object (GS_FLAG_LOAD_RT from the second on) and gs_composite.
 *   assets          [object_count][local_count]: object k's asset on local member i is assets[k * local_count + i]
 *                   (each uploaded with gs_group_asset_upload; an asset may appear in one object only);
 *   fps, do_sort    [object_count]: each object's uniforms (transform, knobs, bits, cutouts, scene depth) and its
 *                   m_FrameCounter % m_SortNthFrame == 0.  All objects must share screen_w / screen_h;
 *   opt             blend_mode and GS_FLAG_ASYNC_READBACK, as gs_group_frame; GS_FLAG_LOAD_RT is refused;
 *   rts             as gs_group_frame;
 *   camera_targets  [local_count], may be NULL or hold NULLs: member i's camera target (host, device or CUDA-array memory,
 *                   width x height) receives the composite pass of the assembled frame, on the member's transfer stream after
 *                   the row exchange.  A device or array target is complete after gs_group_sync (or before the next call's
 *                   draw touches the image); a host target is complete when the call returns.  gs_sync on a member's
 *                   context also waits for that member's composite onto a CUDA-array camera target.
 * Per call: each object is sorted with its own splitters, slab table and order exchange (its order persists in its asset);
 * all objects' distance kernels and view-calcs are queued first and the host waits once for all slab tables.  Each object
 * blends under the earlier ones on the member's own rows; there is ONE row split (balanced on the summed measured cost of the
 * objects) and ONE row exchange per call.  A truncated bin list of any object is reported, as for gs_frame (see "Bin-list
 * capacity"), even when a later object's list fits.  After gs_group_join only the first object ever sorted on the group uses the
 * peer-to-peer order exchange; the others use the all-gather or in-place exchange.  GsGroupStats of such a call: the times
 * span the whole call (slab_sort_ms runs to the end of the last object's slab sort, order_exchange_ms is its exchange,
 * bin_ms sums every object's binning); slab_counts are summed over the objects the call sorted.
 * GS_ERR_INVALID_ARGUMENT, with nothing written: a NULL group / assets / fps / do_sort, object_count 0, a NULL asset, one
 * asset listed for two objects, members of one object holding different splat counts, objects of different screen sizes,
 * GS_FLAG_LOAD_RT, or an image / camera target of the wrong size (bad formats: the image errors of gs_frame).
 * gs_group_frame is this call with one object and no camera targets.  Collective, as gs_group_frame. */
GS_API int gs_group_frame_objects(GsGroup *group, uint32_t object_count, GsAsset *const *assets, const GsFrameParams *fps,
                                  const int32_t *do_sort, const GsRenderOptions *opt, GsImage *const *rts,
                                  GsImage *const *camera_targets);
GS_API int gs_group_sync(GsGroup *group);
GS_API int gs_group_get_stats(GsGroup *group, GsGroupStats *out);
/* The row balancer by itself (host arithmetic, no GPU): splits `rows` 16-pixel rows with the given measured costs into
 * `parts` contiguous ranges of near-equal cost; bounds_out[parts + 1], bounds_out[0] = 0, bounds_out[parts] = rows. */
GS_API int gs_group_balance_rows(const uint32_t *row_cost, uint32_t rows, uint32_t parts, uint32_t *bounds_out);
/* The per-row costs the last gs_group_frame / gs_group_frame_objects call measured: for every 16-pixel row, the summed
 * raster-tile cost of all the objects it drew.  The row split two calls later is gs_group_balance_rows of this vector.
 * row_cost_out[rows], where rows is the number of 16-pixel rows of that call's screen (else GS_ERR_INVALID_ARGUMENT).  Blocks
 * until the vector is on the host.  GS_ERR_NOT_READY before the first call at the current screen size. */
GS_API int gs_group_row_costs(GsGroup *group, uint32_t *row_cost_out, uint32_t rows);

/* ---- stand-alone sorter (GpuSorting.Dispatch, R/GpuSorting.cs:142-198) ----------- */
/* Stable ascending sort of `count` (uint32 key, uint32 payload) pairs in place in DEVICE
 * buffers keys/payload (KEY_UINT PAYLOAD_UINT SHOULD_ASCEND SORT_PAIRS, R/GpuSorting.cs:115-128). */
GS_API int gs_sort_pairs_device(GsContext *ctx, uint32_t *d_keys, uint32_t *d_payload, uint32_t count);
/* Same through HOST buffers (copies in, sorts, copies out, blocks). */
GS_API int gs_sort_pairs_host(GsContext *ctx, uint32_t *keys, uint32_t *payload, uint32_t count);

/* ---- export (EditExportData, R/GaussianSplatRenderer.cs:936-958 -> CSExportData, S/SplatUtilities.compute:616-669) ---- */
/* Decodes every splat of the uploaded asset back to the INRIA .ply attribute record: n x 62 floats in HOST memory `dst`
 * (pos, nor, f_dc, f_rest channel-major, opacity as logit, log scale, rot wxyz -- the InputSplatData layout,
 * E/Utils/GaussianFileReader.cs:17-26).  nor = (1,1,1) marks a splat the cutouts remove (`cutouts` as in GsFrameParams;
 * may be NULL).  gsa_ply_write (gsplat_asset.h) then writes the file ExportPlyFile writes
 * (E/GaussianSplatRendererEditor.cs:394-445).  The baked variant (bake_transform != 0) is a host pass over these records,
 * gsa_bake_transform (gsplat_asset.h); the device entry point itself returns GS_ERR_UNSUPPORTED_FORMAT for the flag.  Blocks. */
GS_API int gs_export_splats(GsContext *ctx, GsAsset *asset, const GsCutout *cutouts, uint32_t cutout_count,
                            uint32_t bake_transform, void *dst);

/* ---- asset packer on the GPU (CreateAsset, E/GaussianSplatAssetCreator.cs:248-330) ----------------------------------
 * The device twin of gsa_create_asset (include/gsplat_asset.h, the host packer): bounds, Morton reorder, SH palette
 * clustering (mini-batch k-means with k-means++ seeding), chunk quantisation, the format encodes and BC7.  For finite input
 * the five blobs and the bounds are the same bytes the host packer writes.  Input containing NaN or Inf still yields a
 * well-formed asset of the right size, without faulting, but its bytes are not guaranteed to match the host packer's. */

/* InputSplatData (E/Utils/GaussianFileReader.cs:17-26), 62 floats / 248 bytes, after LinearizeData: the same layout as
 * GsaInputSplat of gsplat_asset.h, restated so that this header stands alone. */
typedef struct GsInputSplat {
  float pos[3];
  float nor[3];
  float dc0[3];
  float sh[45]; /* sh1..shF, each rgb */
  float opacity;
  float scale[3];
  float rot[4];
} GsInputSplat;

typedef struct GsPackSizes {   /* byte sizes of the five blobs (the gsa_calc_sizes values) and the colour texture */
  uint64_t pos_bytes, other_bytes, color_bytes, sh_bytes, chunk_bytes;
  uint32_t tex_width, tex_height;
} GsPackSizes;

typedef struct GsPackDesc {
  const GsInputSplat *splats;   /* splat_count records; read only, never modified */
  uint32_t splat_count;
  uint32_t memory;              /* GsMemory: where `splats` lives (device memory must belong to the context's device) */
  uint32_t pos_format, scale_format, color_format, sh_format;   /* GsVectorFormat x2, GsColorFormat, GsSHFormat */
} GsPackDesc;

typedef struct GsPackedAsset {
  void *pos, *other, *color, *sh, *chunks;   /* caller's buffers of gs_pack_sizes bytes each; chunks may be NULL when chunk_bytes is 0 */
  uint32_t memory;                           /* GsMemory of the five buffers */
  uint32_t reserved;
  float bounds_min[3], bounds_max[3];        /* out: position bounds of the input */
} GsPackedAsset;

/* gsa_calc_sizes' arithmetic and rules: GS_ERR_UNSUPPORTED_FORMAT for an unknown format or a clustered SH format with no
 * more splats than palette entries. */
GS_API int gs_pack_sizes(uint32_t splat_count, uint32_t pos_format, uint32_t scale_format, uint32_t color_format,
                         uint32_t sh_format, GsPackSizes *out);
/* Packs desc->splats on the context's device.  blobs_out (may be NULL) receives the blobs in host or device memory;
 * asset_out (may be NULL) receives a ready GsAsset, as gs_asset_upload makes it (draw order reset, blobs in HBM), built
 * without a host copy of the blobs.  At least one of the two must be given.  Blocks until the results are complete. */
GS_API int gs_pack_asset(GsContext *ctx, const GsPackDesc *desc, GsPackedAsset *blobs_out, GsAsset **asset_out);
/* The device twin of gsa_kmeans (gsplat_asset.h): the same means and labels, bit for bit.  Host pointers: data
 * n x dim floats, means_out k x dim, labels_out n.  dim must be 1..128. Blocks. */
GS_API int gs_kmeans(GsContext *ctx, uint32_t dim, const float *data, uint32_t n, uint32_t batch, float passes,
                     float *means_out, uint32_t k, int32_t *labels_out);
/* Counters of the last gs_pack_asset: [0] scale^(1/8) values recomputed on the host because the device's double pow
 * result lay next to a float rounding midpoint (see DESIGN.md), [1] k-means mini-batch iterations, [2] k-means++ rounds. */
GS_API int gs_debug_pack_stats(GsContext *ctx, uint64_t out[4]);

/* ---- test hooks (blocking device->host reads) ----------------------------------- */
GS_API int gs_readback_order(GsAsset *asset, uint32_t *dst);      /* _SplatSortKeys, N words */
GS_API int gs_readback_keys(GsAsset *asset, uint32_t *dst);       /* _SplatSortDistances, N words (sorted after gs_sort) */
GS_API int gs_readback_view(GsAsset *asset, void *dst);           /* _SplatViewData, N x 40 bytes (S/GaussianSplatting.hlsl:610-615) */
GS_API int gs_upload_order(GsAsset *asset, const uint32_t *src);  /* seed a previous-frame order */

/* Diagnostics: with GS_RASTER_STATS=1 in the environment the compositor counts, per frame, [0] warp-batches,
 * [1] warp cull ballots, [2] warp candidates, [3] warp evaluations, [4] pixel blends, [5] list entries x warps. */
GS_API int gs_debug_raster_stats(GsContext *ctx, uint64_t out[8]);
/* Diagnostics: with GS_SORT_PHASES=1 in the environment the depth sort records, per pass and 8192-pair tile, 8 words:
 * %globaltimer ns at [0] tile start, [1] keys landed, [2] prefix resolved, [3] scatter done; [4] look-back status words read and
 * [5] status words summed (max over digits); [6] the tile; [7] CTA << 32 | SM.  Pass p's tile t is at (p * tiles + t) * 8;
 * *tiles = tiles per pass.  Copies min(max_words, 32 * tiles) words of the last depth sort. */
GS_API int gs_debug_sort_phases(GsContext *ctx, uint64_t *out, uint32_t max_words, uint32_t *tiles);

/* ---- Unity render-thread entry (SURVEY 8f N2) -------------------------------------- */
/* Unity executes native GPU work on its render thread through CommandBuffer.IssuePluginEventAndData(func, eventId, data)
 * (the reference records everything into CommandBuffers, R/GaussianSplatRenderer.cs:108-211).  `func` is what
 * gs_unity_get_render_event_func returns (signature of Unity's UnityRenderingEventAndData); `data` points to a
 * GsUnityFrameEvent the managed side keeps alive (pinned) until the command buffer has executed.  The callback runs
 * the requested entry point and stores its GsStatus in `status` -- "log and skip", never a throw across the boundary. */
typedef enum GsUnityEvent {
  GS_UNITY_EVENT_FRAME = 1,   /* gs_frame(ctx, asset, &params, &options, do_sort, has_rt ? &rt : NULL, has_camera_target ? &camera_target : NULL) */
  GS_UNITY_EVENT_SYNC = 2,    /* gs_sync(ctx) */
  GS_UNITY_EVENT_FRAME_OBJECTS = 3,  /* data is a GsUnityFrameObjectsEvent: gs_frame_objects(ctx, object_count, assets, fps,
                                        do_sort, &options, has_rt ? &rt : NULL, has_camera_target ? &camera_target : NULL) */
  GS_UNITY_EVENT_FRAME_CAMERAS = 4,  /* data is a GsUnityFrameCamerasEvent: gs_frame_cameras (below) */
  GS_UNITY_EVENT_GROUP_FRAME_OBJECTS = 5,   /* data is a GsUnityGroupFrameObjectsEvent: gs_group_frame_objects (below) */
  GS_UNITY_EVENT_GROUP_SYNC = 6      /* data is a GsUnityGroupSyncEvent: gs_group_sync(group) */
} GsUnityEvent;

typedef struct GsUnityFrameEvent {
  GsContext *ctx;
  GsAsset *asset;
  GsFrameParams params;
  GsRenderOptions options;
  int32_t do_sort;            /* m_FrameCounter % m_SortNthFrame == 0 */
  int32_t status;             /* out: GsStatus of the call (GS_ERR_NOT_READY until the event has run) */
  uint32_t has_rt, has_camera_target;
  GsImage rt, camera_target;
} GsUnityFrameEvent;

/* One camera's splat objects (GS_UNITY_EVENT_FRAME_OBJECTS).  The three arrays are the managed side's, kept alive (pinned)
 * with the payload until the command buffer has executed. */
typedef struct GsUnityFrameObjectsEvent {
  GsContext *ctx;
  uint32_t object_count, reserved0;
  GsAsset *const *assets;     /* [object_count] */
  const GsFrameParams *fps;   /* [object_count] */
  const int32_t *do_sort;     /* [object_count] */
  GsRenderOptions options;
  int32_t status;             /* out: GsStatus of the call (GS_ERR_NOT_READY until the event has run) */
  uint32_t has_rt, has_camera_target, reserved1;
  GsImage rt, camera_target;
} GsUnityFrameObjectsEvent;

/* The payloads of events 4-6 pass images BY VALUE, in arrays of GsImage: an image whose `data` is NULL is "none" (a NULL rt or
 * camera target of the direct call), and a NULL array pointer is the direct call's NULL array.  A managed GsImage[] is then
 * pinned once, and no payload holds a pointer to pointers.  Every array a payload points to, and every GsArrayLayer /
 * GsArrayRect descriptor an image's `data` (or a GsFrameParams' scene_depth) points to, is borrowed: the managed side keeps
 * it pinned (with the payload itself) until the command buffer has executed.  The library never writes them.
 * Each event runs its entry point on the render thread and stores the GsStatus in `status`, which the managed side sets to
 * GS_ERR_NOT_READY when it records the event; the library leaves it alone until the event runs.  An error is reported in
 * `status` and through gs_last_error of the context named below, with the entry point's own code and text; the callback never
 * throws and never aborts.  The device work of an event is the direct call's, launch for launch.  Unity's render thread may
 * have another CUDA device current: the entry points make their contexts' devices current themselves, and the callback makes
 * no CUDA call of its own, so an event leaves current the device the direct call leaves.  The `reserved` words are 0. */

/* GS_UNITY_EVENT_FRAME_CAMERAS: gs_frame_cameras(ctx, camera_count, object_counts, assets, fps, do_sort, &options, rts',
 * camera_targets') where rts'[c] = &rts[c] (NULL where rts[c].data is NULL), likewise camera_targets' -- e.g. the two eyes
 * of a single-pass-instanced XR eye-texture array drawn into layers 0 and 1 as one camera run (GS_MEM_ARRAY_LAYER), or the
 * tiles of an atlas or light-field quilt (GS_MEM_ARRAY_RECT).  At most GS_UNITY_EVENT_MAX_CAMERAS cameras per event: more is
 * GS_ERR_INVALID_ARGUMENT with nothing enqueued (the callback does not allocate; a host with more views issues one event per
 * GS_UNITY_EVENT_MAX_CAMERAS cameras, whose result is the same, as gs_frame_cameras is defined as its camera loop).  Errors:
 * gs_last_error(ctx). */
#define GS_UNITY_EVENT_MAX_CAMERAS 64u
typedef struct GsUnityFrameCamerasEvent {
  GsContext *ctx;
  uint32_t camera_count, reserved0;
  const uint32_t *object_counts;   /* [camera_count] */
  GsAsset *const *assets;          /* [sum of object_counts], camera-major as in gs_frame_cameras */
  const GsFrameParams *fps;        /* [sum of object_counts] */
  const int32_t *do_sort;          /* [sum of object_counts] */
  GsRenderOptions options;
  const GsImage *rts;              /* [camera_count], by value */
  const GsImage *camera_targets;   /* [camera_count], by value */
  int32_t status;                  /* out: GsStatus of the call (GS_ERR_NOT_READY until the event has run) */
  uint32_t reserved1[3];
} GsUnityFrameCamerasEvent;        /* 112 bytes */

/* GS_UNITY_EVENT_GROUP_FRAME_OBJECTS: gs_group_frame_objects(group, object_count, assets, fps, do_sort, &options, rts',
 * camera_targets'), images as above, one per LOCAL member (gs_group_local_count).  The event is collective, as the call is.
 * It holds Unity's render thread where the call blocks: once for all objects' slab tables when the group has several GPUs and
 * an object sorts (see gs_group_frame_objects), and until the transfer streams are done when an image is in host memory and
 * GS_FLAG_ASYNC_READBACK is not set.
 * Errors: gs_last_error of the group's member-0 context (gs_group_context(group, 0)), whichever member the direct call named. */
typedef struct GsUnityGroupFrameObjectsEvent {
  GsGroup *group;
  uint32_t object_count, reserved0;
  GsAsset *const *assets;          /* [object_count][local_count], as in gs_group_frame_objects */
  const GsFrameParams *fps;        /* [object_count] */
  const int32_t *do_sort;          /* [object_count] */
  GsRenderOptions options;
  const GsImage *rts;              /* [local_count], by value */
  const GsImage *camera_targets;   /* [local_count], by value */
  int32_t status;                  /* out: GsStatus of the call (GS_ERR_NOT_READY until the event has run) */
  uint32_t reserved1[3];
} GsUnityGroupFrameObjectsEvent;   /* 104 bytes */

/* GS_UNITY_EVENT_GROUP_SYNC: gs_group_sync(group); blocks the render thread until every member's streams are done.  Errors:
 * gs_last_error of the member-0 context. */
typedef struct GsUnityGroupSyncEvent {
  GsGroup *group;
  int32_t status;                  /* out: GsStatus of the call (GS_ERR_NOT_READY until the event has run) */
  uint32_t reserved;
} GsUnityGroupSyncEvent;           /* 16 bytes */

typedef void (*GsUnityRenderEventAndDataFunc)(int event_id, void *data);
GS_API GsUnityRenderEventAndDataFunc gs_unity_get_render_event_func(void);
GS_API uint32_t gs_unity_frame_event_size(void);   /* sizeof(GsUnityFrameEvent), for the managed side's layout check */
GS_API uint32_t gs_unity_frame_objects_event_size(void);   /* sizeof(GsUnityFrameObjectsEvent) */
GS_API uint32_t gs_unity_frame_cameras_event_size(void);   /* sizeof(GsUnityFrameCamerasEvent) */
GS_API uint32_t gs_unity_group_frame_objects_event_size(void);   /* sizeof(GsUnityGroupFrameObjectsEvent) */
GS_API uint32_t gs_unity_group_sync_event_size(void);   /* sizeof(GsUnityGroupSyncEvent) */

/* ---- device-pointer access for zero-copy hosts (torch / CUDA-Vulkan interop) ----- */
GS_API void *gs_context_stream(GsContext *ctx);
/* 0 order, 1 keys, 2 view (the asset's own); 3 pos, 4 other, 5 sh, 6 color, 7 chunks (NULL when the asset has none): the
 * blobs, the same pointers for an asset and its instances (gs_asset_instance).  Any other `which`: NULL. */
GS_API void *gs_asset_device_ptr(GsAsset *asset, int which);

#ifdef __cplusplus
}
#endif
#endif /* GSPLAT_B200_H */
