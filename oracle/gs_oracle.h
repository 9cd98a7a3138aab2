/* gs_oracle.h -- CPU ORACLE for the Gaussian-splat hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may link or call this.  The product (unitygaussiansplatting_b200/) never does.
 *
 * PINNING: the reference (aras-p/UnityGaussianSplatting @ 2c6fed37) ships no golden
 * vectors, known-answer tests or fixtures for any boundary of this path -- its only goldens
 * are six final PNGs that need the INRIA models, which are not in the repo (SURVEY.md 4, 8c)
 * -- and neither its C# (Unity + Burst) nor its HLSL (DXC + a GPU) runs in this image.
 * What pins this restatement instead is the reference's shader SOURCE ITSELF: oracle/refhlsl/
 * compiles package/Shaders/{GaussianSplatting.hlsl, SplatUtilities.compute, SphericalHarmonics.hlsl,
 * RenderGaussianSplats.shader} where they lie, with g++, against a C++ shim of HLSL's types and
 * intrinsics (oracle/_ref/libref_hlsl.so), and tests/test_reference_hlsl.py compares this file
 * with it stage by stage: sort keys, LoadSplatData + CSCalcViewData, vert + frag, CSExportData
 * incl. RotateSH -- agreement to float rounding (the two evaluate the same formulas under
 * different but equally valid contraction / evaluation orders).  NOT covered by that pin:
 * the fixed-function parts (which pixels a quad covers, the RGBA16F blend), the sort's
 * tie semantics, and UnityCG's GammaToLinearSpace (third party, not in the reference repo);
 * those rest on analytic checks and the published formulas (tests/test_oracle_*.py).
 *
 * Arithmetic contract (shared by design with the CUDA path so both can be compared
 * bit-for-bit; HLSL leaves all of this to the driver compiler, so nothing here is pinned
 * by the reference):
 *   - IEEE float32, no contraction (build with -ffp-contract=off), expressions evaluate
 *     left to right exactly as written; fmaf() only where written.
 *   - "x / K" for the unorm decoders is x * (float)(1.0/K)  (what fxc/dxc emit for a
 *     divide by a literal).
 *   - mul(M, float4(p,1)).i = fmaf(Mi2,z, fmaf(Mi1,y, fmaf(Mi0,x, Mi3))).
 *   - lerp(a,b,t) = fmaf(t, b-a, a).
 *   - normalize(v) = v / sqrt(dot(v,v)); length = sqrt; rcp = 1/x; all IEEE.
 *   - f32tof16 rounds to nearest even; f16tof32 exact.
 *   - exp() in the splat pixel shader is gso_exp_neg(): 2^(x*log2e) by magic-number
 *     range reduction and a fixed degree-5 polynomial (max rel. error 7e-7 on [-8,0], the same
 *     class as a GPU's ex2.approx), so the discard test alpha < 1/255 is reproducible.
 *
 * Citations: S/ = package/Shaders, R/ = package/Runtime of the reference.
 */
#ifndef GS_ORACLE_H
#define GS_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSO_API __attribute__((visibility("default")))

typedef struct GsoAsset {            /* R/GaussianSplatAsset.cs:219-237 */
  uint32_t splat_count;
  uint32_t pos_format, scale_format, sh_format, color_format;
  const void *pos, *other, *sh, *color, *chunks; /* chunks NULL => _SplatChunkCount = 0 */
  uint64_t pos_bytes, other_bytes, sh_bytes, color_bytes, chunk_bytes;
} GsoAsset;

typedef struct GsoCutout { float mat[16]; uint32_t type_and_flags; } GsoCutout;

typedef struct GsoFrame {            /* same fields as GsFrameParams (include/gsplat_b200.h) */
  float mat_object_to_world[16], mat_world_to_object[16], mat_view[16], mat_proj_gpu[16];
  float screen_w, screen_h;
  float cam_pos_world[3];
  float splat_scale, opacity_scale;
  uint32_t sh_order, sh_only;
  uint32_t cutout_count, reserved0;
  const GsoCutout *cutouts;
  const uint32_t *deleted_bits;
  const uint32_t *selected_bits;     /* _SplatSelectedBits: read by the splat VERTEX shader, S/RenderGaussianSplats.shader:63-73 */
  const float *scene_depth;          /* the camera's depth buffer the splat pass tests against (ZTest LEqual, ZWrite Off), W x H, reversed Z */
  uint32_t scene_depth_on_device, reserved1;
} GsoFrame;

typedef struct GsoSplat {            /* SplatData, S/GaussianSplatting.hlsl:209-216 */
  float pos[3];
  float rot[4];
  float scale[3];
  float opacity;
  float col[3];
  float sh[45];                      /* sh1..sh15 rgb */
} GsoSplat;

typedef struct GsoView {             /* SplatViewData, S/GaussianSplatting.hlsl:610-615 (40 bytes) */
  float pos[4];
  float axis1[2], axis2[2];
  uint32_t color[2];
} GsoView;

/* ---- scalar helpers (exposed for tests) ---- */
GSO_API uint32_t gso_f32tof16(float f);          /* RNE */
GSO_API float gso_f16tof32(uint32_t h);
GSO_API float gso_exp_neg(float x);              /* deterministic exp for the pixel shader */
GSO_API uint32_t gso_float_to_sortable_uint(float f);  /* S/SplatUtilities.compute:52-57 */
GSO_API float gso_inv_square_centered01(float x);      /* S/GaussianSplatting.hlsl:5-11 */
/* BC7 (BPTC) block -> 16 RGBA8 pixels in raster order; what the texture unit does for ColorFormat.BC7 (R/GaussianSplatAsset.cs:169) */
GSO_API void gso_bc7_decode_block(const uint8_t block[16], uint8_t out_rgba[64]);
GSO_API uint32_t gso_splat_index_to_pixel_index(uint32_t idx, uint32_t *x, uint32_t *y); /* :183-194 */

/* ---- decode (LoadSplatData / LoadSplatPos, S/GaussianSplatting.hlsl:394-421,428-608) ---- */
GSO_API void gso_load_splat_pos(const GsoAsset *a, uint32_t idx, float out[3]);
GSO_API void gso_load_splat_data(const GsoAsset *a, uint32_t idx, GsoSplat *out);

/* ---- CSSetIndices / CSCalcDistances (S/SplatUtilities.compute:59-82; uniforms
 *      R/GaussianSplatRenderer.cs:612-633).  keys[i] = key(pos[order[i]]). ---- */
GSO_API void gso_set_indices(uint32_t *order, uint32_t n);
GSO_API void gso_calc_distances(const GsoAsset *a, const GsoFrame *f, const uint32_t *order, uint32_t *keys,
                                int threads);

/* ---- GpuSorting.Dispatch semantics (R/GpuSorting.cs:142-198; S/DeviceRadixSort.hlsl):
 *      stable ascending sort of (key, payload) pairs, 8-bit LSD, 4 passes, in place. ---- */
GSO_API void gso_sort_pairs(uint32_t *keys, uint32_t *payload, uint32_t n, int threads);

/* ---- CSCalcViewData (S/SplatUtilities.compute:189-252) ---- */
GSO_API void gso_calc_view(const GsoAsset *a, const GsoFrame *f, GsoView *view, int threads);

/* ---- CSExportData (S/SplatUtilities.compute:616-669, no baked transform): n x 62 floats, the .ply attribute record; f may be NULL ---- */
GSO_API void gso_export_data(const GsoAsset *a, const GsoFrame *f, float *out62, int threads);

/* ---- DrawProcedural of RenderGaussianSplats.shader (S/RenderGaussianSplats.shader:35-108,
 *      blend :10-12) into a cleared RT.  rt: W*H*4 floats, premultiplied RGBA; with
 *      blend_mode 0 (fp16 ROP) every value is exactly representable in half. ---- */
GSO_API void gso_render(const GsoView *view, const uint32_t *order, uint32_t n, uint32_t width, uint32_t height,
                        uint32_t blend_mode, float *rt, int threads);
/* The same draw with the edit selection: a splat whose bit is set leaves the vertex shader with col.a = -1 (:63-73) and takes
 * the pixel shader's "selected" branch (:87-101).  selected_bits NULL == _SplatBitsValid 0 == gso_render. */
GSO_API void gso_render_sel(const GsoView *view, const uint32_t *order, uint32_t n, uint32_t width, uint32_t height,
                        uint32_t blend_mode, float *rt, int threads, const uint32_t *selected_bits);
/* ... and with the scene's depth buffer bound (R/GaussianSplatRenderer.cs:195 binds the current depth target; the pass keeps
 * ShaderLab's default ZTest LEqual, ZWrite Off, S/RenderGaussianSplats.shader:8-12).  A splat's quad is flat: every fragment
 * has the depth clip.z / clip.w of the centre.  `scene_depth` is W x H float32 in the GPU projection's convention (reversed Z:
 * 1 = near), under which LEqual is evaluated as "fragment depth >= stored depth".  NULL = no test.  load != 0: the draw starts
 * from rt as given instead of clearing it (GS_FLAG_LOAD_RT: a target earlier draws or the host filled); a pixel no fragment
 * blends into keeps its bits, and a blend that yields NaN stores the GPU's canonical NaN 0x7FFFFFFF (in either blend mode). */
GSO_API void gso_render_ex(const GsoView *view, const uint32_t *order, uint32_t n, uint32_t width, uint32_t height,
                        uint32_t blend_mode, float *rt, int threads, const uint32_t *selected_bits, const float *scene_depth,
                        int load);

/* ---- GaussianComposite.shader:35-39, Blend SrcAlpha OneMinusSrcAlpha (:11).
 *      target: W*H*4 floats, read-modify-write; target_fp16 != 0 rounds the result to half. ---- */
GSO_API void gso_composite(const float *rt, float *target, uint32_t width, uint32_t height, int target_fp16);

GSO_API int gso_max_threads(void);

#ifdef __cplusplus
}
#endif
#endif
