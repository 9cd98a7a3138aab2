// GaussianSplatNativeFrame.cs -- Unity-side shim for libgsplat_b200 (SURVEY 8f row N2).
//
// NOT compiled or run in this repository (no Unity / dotnet toolchain in the build image): it is the file a maintainer
// drops next to package/Runtime/GaussianSplatRenderer.cs, together with GaussianSplatNative.cs from INTEGRATION.md.
// What it replaces: the per-renderer body of GaussianSplatRenderSystem.SortAndRenderSplats
// (package/Runtime/GaussianSplatRenderer.cs:118-166: SortPoints + CalcViewData + DrawProcedural) by ONE native event on
// Unity's render thread.  The native side of the event (gs_unity_get_render_event_func, GsUnityFrameEvent in
// include/gsplat_b200.h) is built and tested here (tests/test_zz_unity_event.py).  GaussianSplatNativeCameraFrame below
// records ONE event for all of a camera's active splat objects (GS_UNITY_EVENT_FRAME_OBJECTS -> gs_frame_objects; tested in
// tests/test_gpu_frame_objects.py).
using System;
using System.Collections.Generic;
using System.Runtime.InteropServices;
using Unity.Collections;
using Unity.Collections.LowLevel.Unsafe;
using UnityEngine;
using UnityEngine.Rendering;

namespace GaussianSplatting.Runtime
{
    /// One of these per GaussianSplatRenderer; owns the pinned event payloads handed to the render thread.
    internal sealed unsafe class GaussianSplatNativeFrame : IDisposable
    {
        [StructLayout(LayoutKind.Sequential)]
        struct GsUnityFrameEvent                                    // include/gsplat_b200.h (size checked against gs_unity_frame_event_size)
        {
            public IntPtr ctx, asset;
            public GaussianSplatNative.GsFrameParams fp;
            public GaussianSplatNative.GsRenderOptions options;
            public int do_sort, status;
            public uint has_rt, has_camera_target;
            public GaussianSplatNative.GsImage rt, camera_target;
        }

        // include/gsplat_b200.h: a rectangle of a 2-D CUDA array or of one layer of a layered one (GS_MEM_ARRAY_RECT = 5), 24 bytes
        [StructLayout(LayoutKind.Sequential)]
        internal struct GsArrayRect
        {
            public IntPtr array;
            public uint layer, x, y, reserved;
        }

        [DllImport("gsplat_b200")] static extern IntPtr gs_unity_get_render_event_func();
        [DllImport("gsplat_b200")] static extern uint gs_unity_frame_event_size();

        const int kEventFrame = 1;                                  // GS_UNITY_EVENT_FRAME
        internal const int kInFlight = 3;                                   // command buffers may execute up to 2 frames late
        NativeArray<GsUnityFrameEvent> m_Events;                    // persistent => stable address, no GC pinning needed
        NativeArray<GsArrayRect> m_Rects;                           // each slot's rt rectangle (RecordRect), borrowed until its event has run
        // The reference binds _SplatCutouts / _SplatDeletedBits / _SplatSelectedBits on every CalcViewData (SetAssetDataOnCS,
        // R/GaussianSplatRenderer.cs:485-509).  The native frame takes them as HOST arrays borrowed until the event has run,
        // so every in-flight slot owns its copies.  The bit arrays live in GraphicsBuffers in the reference (edited by compute
        // kernels); a host that edits must keep a CPU mirror of them (hostDeletedBits / hostSelectedBits below) -- without
        // one, pass default and the frame renders as if nothing were deleted or selected.
        NativeArray<GaussianCutout.ShaderData>[] m_Cutouts = new NativeArray<GaussianCutout.ShaderData>[kInFlight];
        NativeArray<uint>[] m_Deleted = new NativeArray<uint>[kInFlight], m_Selected = new NativeArray<uint>[kInFlight];
        int m_Next;
        internal static readonly IntPtr s_EventFunc = gs_unity_get_render_event_func();

        public GaussianSplatNativeFrame()
        {
            if (gs_unity_frame_event_size() != (uint)UnsafeUtility.SizeOf<GsUnityFrameEvent>())
                throw new InvalidOperationException("GsUnityFrameEvent layout mismatch between C# and libgsplat_b200");
            m_Events = new NativeArray<GsUnityFrameEvent>(kInFlight, Allocator.Persistent);
            m_Rects = new NativeArray<GsArrayRect>(kInFlight, Allocator.Persistent);
        }

        public void Dispose()
        {
            if (m_Events.IsCreated) m_Events.Dispose();
            if (m_Rects.IsCreated) m_Rects.Dispose();
            for (int i = 0; i < kInFlight; ++i)
            {
                if (m_Cutouts[i].IsCreated) m_Cutouts[i].Dispose();
                if (m_Deleted[i].IsCreated) m_Deleted[i].Dispose();
                if (m_Selected[i].IsCreated) m_Selected[i].Dispose();
            }
        }

        static void CopyInto<T>(ref NativeArray<T> dst, NativeArray<T> src) where T : unmanaged
        {
            if (!dst.IsCreated || dst.Length != src.Length)
            {
                if (dst.IsCreated) dst.Dispose();
                dst = new NativeArray<T>(src.Length, Allocator.Persistent, NativeArrayOptions.UninitializedMemory);
            }
            dst.CopyFrom(src);
        }


        /// Records the native frame into `cmb`.  `rtArray` is the cudaArray_t of _GaussianSplatRT's R16G16B16A16_SFloat image
        /// that the graphics-interop plugin imported (cudaImportExternalMemory -> cudaExternalMemoryGetMappedMipmappedArray with
        /// cudaArraySurfaceLoadStore -> cudaGetMipmappedArrayLevel 0; INTEGRATION.md section 3).  The library renders into it in
        /// place; the composite draw that follows in the reference (:206-210) stays as it is and samples that texture.
        public void Record(CommandBuffer cmb, GaussianSplatRenderer gs, Camera cam, IntPtr ctx, IntPtr asset, IntPtr rtArray,
                           int rtWidth, int rtHeight, NativeArray<uint> hostDeletedBits = default, NativeArray<uint> hostSelectedBits = default)
        {
            // results of the event recorded kInFlight frames ago: log and skip, like the reference (:655)
            var ev = (GsUnityFrameEvent*)m_Events.GetUnsafePtr() + m_Next;
            if (ev->ctx != IntPtr.Zero && ev->status != 0 && ev->status != -5)
                GaussianSplatNative.Check(ev->ctx, ev->status);

            ev->ctx = ctx;
            ev->asset = asset;
            ev->fp = FillParams(m_Next, gs, cam, rtWidth, rtHeight, hostDeletedBits, hostSelectedBits);
            ev->options = default;                                                    // fp16-ROP blend, whole image
            ev->do_sort = gs.m_FrameCounter % gs.m_SortNthFrame == 0 ? 1 : 0;         // :120-121
            ev->status = -5;                                                          // GS_ERR_NOT_READY until it has run
            ev->has_rt = 1; ev->has_camera_target = 0;
            ev->rt = new GaussianSplatNative.GsImage
            {
                data = (void*)rtArray, width = (uint)rtWidth, height = (uint)rtHeight,
                row_pitch_bytes = 0, format = 0 /* GS_PIX_RGBA16F */, memory = 2 /* GS_MEM_ARRAY */
            };
            ++gs.m_FrameCounter;
            cmb.IssuePluginEventAndData(s_EventFunc, kEventFrame, (IntPtr)ev);
            m_Next = (m_Next + 1) % kInFlight;
        }

        /// As Record, into the rtWidth x rtHeight rectangle at the origin of a larger texture: HDRP's _GaussianSplatRT is an
        /// RTHandle allocated at the largest size any camera has needed (INTEGRATION.md section 3, "HDRP"), and the camera draws
        /// into its scaled pixel size at texel (0, 0).  `rtArray` is that texture's import, redone when the RTHandle grows.
        public void RecordRect(CommandBuffer cmb, GaussianSplatRenderer gs, Camera cam, IntPtr ctx, IntPtr asset, IntPtr rtArray,
                               int rtWidth, int rtHeight, NativeArray<uint> hostDeletedBits = default, NativeArray<uint> hostSelectedBits = default)
        {
            int slot = m_Next;
            var rect = (GsArrayRect*)m_Rects.GetUnsafePtr() + slot;
            *rect = new GsArrayRect { array = rtArray, layer = 0, x = 0, y = 0, reserved = 0 };
            Record(cmb, gs, cam, ctx, asset, rtArray, rtWidth, rtHeight, hostDeletedBits, hostSelectedBits);
            var ev = (GsUnityFrameEvent*)m_Events.GetUnsafePtr() + slot;
            ev->rt.data = rect;
            ev->rt.memory = 5;   // GS_MEM_ARRAY_RECT; the event has been recorded, but it reads its payload only when it runs
        }

        /// The renderer's uniforms for in-flight slot `slot`.  The cutouts and bits they point to are this object's copies for
        /// that slot, alive until the slot is used again kInFlight events later.
        internal GaussianSplatNative.GsFrameParams FillParams(int slot, GaussianSplatRenderer gs, Camera cam, int rtWidth, int rtHeight,
                                                              NativeArray<uint> hostDeletedBits, NativeArray<uint> hostSelectedBits)
        {
            var tr = gs.transform;
            var fp = new GaussianSplatNative.GsFrameParams
            {
                mat_object_to_world = tr.localToWorldMatrix,
                mat_world_to_object = tr.worldToLocalMatrix,
                mat_view = cam.worldToCameraMatrix,
                mat_proj_gpu = GL.GetGPUProjectionMatrix(cam.projectionMatrix, true),   // UNITY_MATRIX_P is an engine global
                screen_w = rtWidth, screen_h = rtHeight,
                cam_pos_world = cam.transform.position,
                splat_scale = gs.m_SplatScale, opacity_scale = gs.m_OpacityScale,
                sh_order = (uint)gs.m_SHOrder, sh_only = gs.m_SHOnly ? 1u : 0u,
            };
            // cutouts: the ShaderData records UpdateCutoutsBuffer builds (R/GaussianSplatRenderer.cs:511-531), matrix = cutout
            // worldToLocal * renderer localToWorld (R/GaussianCutout.cs:26-40)
            fp.cutouts = null; fp.cutout_count = 0; fp.deleted_bits = null; fp.selected_bits = null;
            if (gs.m_Cutouts != null && gs.m_Cutouts.Length > 0)
            {
                var data = new NativeArray<GaussianCutout.ShaderData>(gs.m_Cutouts.Length, Allocator.Temp);
                for (int i = 0; i < gs.m_Cutouts.Length; ++i) data[i] = GaussianCutout.GetShaderData(gs.m_Cutouts[i], tr.localToWorldMatrix);
                CopyInto(ref m_Cutouts[slot], data);
                data.Dispose();
                fp.cutouts = (GaussianCutout.ShaderData*)m_Cutouts[slot].GetUnsafePtr();
                fp.cutout_count = (uint)m_Cutouts[slot].Length;
            }
            int words = (gs.splatCount + 31) / 32;
            if (hostDeletedBits.IsCreated && hostDeletedBits.Length >= words)
            {
                CopyInto(ref m_Deleted[slot], hostDeletedBits);
                fp.deleted_bits = (uint*)m_Deleted[slot].GetUnsafePtr();
            }
            if (hostSelectedBits.IsCreated && hostSelectedBits.Length >= words)
            {
                CopyInto(ref m_Selected[slot], hostSelectedBits);
                fp.selected_bits = (uint*)m_Selected[slot].GetUnsafePtr();
            }
            return fp;
        }
    }

    /// One per camera: the camera's active splat objects, in GatherSplatsForCamera order, drawn by ONE native event
    /// (GS_UNITY_EVENT_FRAME_OBJECTS -> gs_frame_objects): _GaussianSplatRT cleared once, one bin list and one raster for all
    /// of them, instead of one event per object.  Each object keeps its GaussianSplatNativeFrame for its cutout and bit
    /// copies; every asset must live on `ctx`.
    internal sealed unsafe class GaussianSplatNativeCameraFrame : IDisposable
    {
        [StructLayout(LayoutKind.Sequential)]
        struct GsUnityFrameObjectsEvent                             // include/gsplat_b200.h (size checked against gs_unity_frame_objects_event_size)
        {
            public IntPtr ctx;
            public uint object_count, reserved0;
            public IntPtr* assets;
            public GaussianSplatNative.GsFrameParams* fps;
            public int* do_sort;
            public GaussianSplatNative.GsRenderOptions options;
            public int status;
            public uint has_rt, has_camera_target, reserved1;
            public GaussianSplatNative.GsImage rt, camera_target;
        }

        [DllImport("gsplat_b200")] static extern uint gs_unity_frame_objects_event_size();

        const int kEventFrameObjects = 3;                           // GS_UNITY_EVENT_FRAME_OBJECTS
        const int kInFlight = GaussianSplatNativeFrame.kInFlight;
        NativeArray<GsUnityFrameObjectsEvent> m_Events;
        // what each in-flight event points to: the library reads these arrays on the render thread
        NativeArray<IntPtr>[] m_Assets = new NativeArray<IntPtr>[kInFlight];
        NativeArray<GaussianSplatNative.GsFrameParams>[] m_Params = new NativeArray<GaussianSplatNative.GsFrameParams>[kInFlight];
        NativeArray<int>[] m_DoSort = new NativeArray<int>[kInFlight];
        int m_Next;

        public GaussianSplatNativeCameraFrame()
        {
            if (gs_unity_frame_objects_event_size() != (uint)UnsafeUtility.SizeOf<GsUnityFrameObjectsEvent>())
                throw new InvalidOperationException("GsUnityFrameObjectsEvent layout mismatch between C# and libgsplat_b200");
            m_Events = new NativeArray<GsUnityFrameObjectsEvent>(kInFlight, Allocator.Persistent);
        }

        public void Dispose()
        {
            if (m_Events.IsCreated) m_Events.Dispose();
            for (int i = 0; i < kInFlight; ++i)
            {
                if (m_Assets[i].IsCreated) m_Assets[i].Dispose();
                if (m_Params[i].IsCreated) m_Params[i].Dispose();
                if (m_DoSort[i].IsCreated) m_DoSort[i].Dispose();
            }
        }

        static void Ensure<T>(ref NativeArray<T> a, int n) where T : unmanaged
        {
            if (a.IsCreated && a.Length == n) return;
            if (a.IsCreated) a.Dispose();
            a = new NativeArray<T>(n, Allocator.Persistent, NativeArrayOptions.UninitializedMemory);
        }

        /// Records the camera's frame into `cmb`: `active` in GatherSplatsForCamera order (R/GaussianSplatRenderer.cs:73-105), each
        /// object with its storage and its asset on `ctx`; `rtArray` as in GaussianSplatNativeFrame.Record.  The composite draw
        /// that follows in the reference (:206-210) stays as it is.
        public void Record(CommandBuffer cmb, List<(GaussianSplatRenderer gs, GaussianSplatNativeFrame storage, IntPtr asset)> active,
                           Camera cam, IntPtr ctx, IntPtr rtArray, int rtWidth, int rtHeight)
        {
            if (active.Count == 0) return;   // no active splat object: OnPreCullCamera draws nothing
            var ev = (GsUnityFrameObjectsEvent*)m_Events.GetUnsafePtr() + m_Next;
            if (ev->ctx != IntPtr.Zero && ev->status != 0 && ev->status != -5)
                GaussianSplatNative.Check(ev->ctx, ev->status);
            int slot = m_Next, n = active.Count;
            Ensure(ref m_Assets[slot], n);
            Ensure(ref m_Params[slot], n);
            Ensure(ref m_DoSort[slot], n);
            for (int i = 0; i < n; ++i)
            {
                var (gs, storage, asset) = active[i];
                m_Assets[slot][i] = asset;
                m_Params[slot][i] = storage.FillParams(slot, gs, cam, rtWidth, rtHeight, default, default);
                m_DoSort[slot][i] = gs.m_FrameCounter % gs.m_SortNthFrame == 0 ? 1 : 0;   // :120-121
                ++gs.m_FrameCounter;
            }
            ev->ctx = ctx;
            ev->object_count = (uint)n;
            ev->assets = (IntPtr*)m_Assets[slot].GetUnsafePtr();
            ev->fps = (GaussianSplatNative.GsFrameParams*)m_Params[slot].GetUnsafePtr();
            ev->do_sort = (int*)m_DoSort[slot].GetUnsafePtr();
            ev->options = default;                                  // fp16-ROP blend, whole image; the call clears the target once
            ev->status = -5;                                        // GS_ERR_NOT_READY until it has run
            ev->has_rt = 1; ev->has_camera_target = 0;
            ev->rt = new GaussianSplatNative.GsImage
            {
                data = (void*)rtArray, width = (uint)rtWidth, height = (uint)rtHeight,
                row_pitch_bytes = 0, format = 0 /* GS_PIX_RGBA16F */, memory = 2 /* GS_MEM_ARRAY */
            };
            cmb.IssuePluginEventAndData(GaussianSplatNativeFrame.s_EventFunc, kEventFrameObjects, (IntPtr)ev);
            m_Next = (m_Next + 1) % kInFlight;
        }
    }
    /// The camera's colour buffer as a camera target (GsImage) of an event, e.g. GsUnityFrameEvent.camera_target with
    /// has_camera_target = 1: URP's HDR camera colour (m_HDRColorBufferPrecision 32-bit, no alpha) and HDRP's
    /// ctx.cameraColorBuffer (colorBufferFormat R11G11B10) are GraphicsFormat.B10G11R11_UFloatPack32, which the library
    /// composites onto in place as GS_PIX_B10G11R11_UFLOAT (2); the built-in pipeline's ARGBHalf is GS_PIX_RGBA16F (0).  An
    /// LDR camera (HDR off) in a linear-colour-space project, and the validator's RenderTexture, draw into
    /// GraphicsFormat.R8G8B8A8_SRGB, which is GS_PIX_R8G8B8A8_SRGB (3).
    /// `colorArray` is the buffer imported as a CUDA array: for B10G11R11 with ONE 32-bit unsigned channel
    /// (cudaCreateChannelDesc<unsigned int>()), for R8G8B8A8_SRGB with FOUR 8-bit unsigned channels
    /// (cudaCreateChannelDesc<uchar4>(); INTEGRATION.md section 3).  Not compiled here, like the rest of this file.
    internal static class GaussianSplatCameraTarget
    {
        public static uint PixelFormat(UnityEngine.Experimental.Rendering.GraphicsFormat f)
        {
            switch (f)
            {
                case UnityEngine.Experimental.Rendering.GraphicsFormat.R16G16B16A16_SFloat: return 0;   // GS_PIX_RGBA16F
                case UnityEngine.Experimental.Rendering.GraphicsFormat.R32G32B32A32_SFloat: return 1;   // GS_PIX_RGBA32F
                case UnityEngine.Experimental.Rendering.GraphicsFormat.B10G11R11_UFloatPack32: return 2; // GS_PIX_B10G11R11_UFLOAT
                case UnityEngine.Experimental.Rendering.GraphicsFormat.R8G8B8A8_SRGB: return 3;          // GS_PIX_R8G8B8A8_SRGB
                default: throw new NotSupportedException("camera colour format " + f + " is not a supported camera target");
            }
        }

        public static unsafe GaussianSplatNative.GsImage Image(IntPtr colorArray, int width, int height,
                                                               UnityEngine.Experimental.Rendering.GraphicsFormat f)
        {
            return new GaussianSplatNative.GsImage
            {
                data = (void*)colorArray, width = (uint)width, height = (uint)height,
                row_pitch_bytes = 0, format = PixelFormat(f), memory = 2 /* GS_MEM_ARRAY */
            };
        }
    }
}
