// AmbientOcclusionNative.cs -- the C# host a MiniEngineAO maintainer would drop next to
// Assets/MiniEngineAO/AmbientOcclusion.cs to route the compute path through libmeao (include/meao.h).
//
// SOURCE ONLY: this image has no C# toolchain (dotnet / mono / mcs / csc are absent, SURVEY.md 8c), so
// this file is neither compiled nor tested here; the Python host miniengineao_b200/ambient_occlusion.py
// is its executable twin and exercises exactly the same entry points.
//
// What changes relative to the reference component:
//   * the parameter surface (AmbientOcclusion.cs:20-68), CheckPropertiesChanged (:104-113) and the
//     LateUpdate re-plan triggers (:329-350) are kept verbatim in spirit;
//   * PushDownsampleCommands / PushRenderCommands x4 / PushUpsampleCommands x4 (:604-785) are replaced
//     by ONE CommandBuffer.IssuePluginEvent that replays libmeao's captured CUDA graph;
//   * texture interop (D3D <-> CUDA) is engine specific and out of scope: the plugin consumes / produces
//     linear device buffers (cudaGraphicsD3D11RegisterResource would map the depth and AO textures).

using System;
using System.Runtime.InteropServices;
using UnityEngine;
using UnityEngine.Rendering;

namespace MiniEngineAO
{
    internal static class MeaoNative
    {
        const string Lib = "meao";   // libmeao.so / meao.dll

        [StructLayout(LayoutKind.Sequential)]
        public struct MeaoParams
        {
            public float noise_filter_tolerance, blur_tolerance, upsample_tolerance, thickness_modifier, intensity;
            public int debug, ambient_only;
        }

        [StructLayout(LayoutKind.Sequential)]
        public struct MeaoCamera
        {
            public float near_clip, far_clip, tan_half_fov_h;
            public int reversed_z;
        }

        [StructLayout(LayoutKind.Sequential)]
        public struct MeaoDeviceCfg { public int device; public uint flags; }

        // Variants the reference ships in its shaders but never selects (meao.h: MeaoVariants); all zero = reference behaviour.
        [StructLayout(LayoutKind.Sequential)]
        public struct MeaoVariants { public int single_pass_stereo, sample_exhaustively, high_quality_mask, single_scale; }

        [DllImport(Lib)] public static extern int meao_create(ref MeaoDeviceCfg cfg, out IntPtr ctx);
        [DllImport(Lib)] public static extern void meao_destroy(IntPtr ctx);
        [DllImport(Lib)] public static extern IntPtr meao_last_error(IntPtr ctx);
        [DllImport(Lib)] public static extern int meao_set_params(IntPtr ctx, ref MeaoParams p);
        [DllImport(Lib)] public static extern int meao_set_variants(IntPtr ctx, ref MeaoVariants v);
        [DllImport(Lib)] public static extern int meao_set_camera(IntPtr ctx, ref MeaoCamera c);
        [DllImport(Lib)] public static extern int meao_resize(IntPtr ctx, int width, int height);
        // Dynamic resolution: what meao_reservation reports (meao.h MeaoReservation)
        [StructLayout(LayoutKind.Sequential)]
        public struct MeaoReservation
        {
            public int width, height;
            public long arena_bytes, arena_bytes_needed, arena_allocations, graphs_held, graph_instantiations;
        }
        // lay the intermediates out once for the largest size; a resize inside it then allocates and synchronises nothing (0, 0 clears)
        [DllImport(Lib)] public static extern int meao_reserve(IntPtr ctx, int maxWidth, int maxHeight);
        [DllImport(Lib)] public static extern int meao_reservation(IntPtr ctx, out MeaoReservation r);
        [DllImport(Lib)] public static extern int meao_set_layers(IntPtr ctx, int layers);   // layered frames: L views per frame, [L][H][W] buffers
        // one camera per layer (split-screen viewports, mirrors, batches from several cameras); null with count 0 clears the table
        [DllImport(Lib)] public static extern int meao_set_layer_cameras(IntPtr ctx, [In] MeaoCamera[] cameras, int count);
        [DllImport(Lib)] public static extern int meao_get_layer_cameras(IntPtr ctx, [Out] MeaoCamera[] cameras, int capacity);
        [DllImport(Lib)] public static extern int meao_render(IntPtr ctx, IntPtr depthDev, int depthKind, IntPtr aoOutDev, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_render_host(IntPtr ctx, float[] depth, int depthKind, byte[] aoOut);
        [DllImport(Lib)] public static extern int meao_bind_event(IntPtr ctx, int eventId, IntPtr depthDev, int depthKind, IntPtr aoOutDev, IntPtr stream);
        // CUDA arrays (graphics interop: cudaGraphicsSubResourceGetMappedArray / level 0 of a Vulkan mipmapped array), no copies
        [DllImport(Lib)] public static extern int meao_render_arrays(IntPtr ctx, IntPtr depthArray, int depthKind, IntPtr aoArray, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_bind_event_arrays(IntPtr ctx, int eventId, IntPtr depthArray, int depthKind, IntPtr aoArray, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_release_array(IntPtr ctx, IntPtr array);   // before the array is unmapped / unregistered / freed
        // Linear buffers with their own row and layer pitch, in bytes (D3D12 placed footprints, Vulkan buffers through external memory,
        // cudaMallocPitch, a dynamic-resolution corner of a max-size target), no copies
        [DllImport(Lib)] public static extern int meao_render_pitched(IntPtr ctx, IntPtr depthDev, long depthRowPitch, long depthLayerPitch, int depthKind,
                                                                      IntPtr aoOutDev, long aoRowPitch, long aoLayerPitch, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_bind_event_pitched(IntPtr ctx, int eventId, IntPtr depthDev, long depthRowPitch, long depthLayerPitch,
                                                                          int depthKind, IntPtr aoOutDev, long aoRowPitch, long aoLayerPitch, IntPtr stream);
        [DllImport(Lib)] public static extern IntPtr meao_get_render_event_func();
        [DllImport(Lib)] public static extern int meao_composite_framebuffer(IntPtr ctx, IntPtr aoDev, IntPtr colorDev, int colorFormat, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_composite_gbuffer(IntPtr ctx, IntPtr aoDev, IntPtr gbuffer0Dev, IntPtr gbuffer3Dev, int gbuffer3Format, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_composite_debug(IntPtr ctx, IntPtr viewR8Dev, IntPtr colorDev, int colorFormat, IntPtr stream);   // AO.cs:826-829
        [DllImport(Lib)] public static extern int meao_get_buffer(IntPtr ctx, int bufferId, IntPtr hostOut, UIntPtr hostBytes);
        [DllImport(Lib)] public static extern int meao_debug_view(IntPtr ctx, int bufferId, IntPtr outR8Dev, IntPtr stream);   // AO.cs:787-820

        public static void Check(IntPtr ctx, int rc)
        {
            if (rc < 0) throw new InvalidOperationException("libmeao: " + Marshal.PtrToStringAnsi(meao_last_error(ctx)));
        }
    }

    [ExecuteInEditMode]
    [RequireComponent(typeof(Camera))]
    public sealed class AmbientOcclusionNative : MonoBehaviour
    {
        // ---- exposed properties: same names, ranges and defaults as AmbientOcclusion.cs:20-68 ----
        [SerializeField, Range(-8, 0)] float _noiseFilterTolerance = 0;
        public float noiseFilterTolerance { get { return _noiseFilterTolerance; } set { _noiseFilterTolerance = value; } }

        [SerializeField, Range(-8, -1)] float _blurTolerance = -4.6f;
        public float blurTolerance { get { return _blurTolerance; } set { _blurTolerance = value; } }

        [SerializeField, Range(-12, -1)] float _upsampleTolerance = -12;
        public float upsampleTolerance { get { return _upsampleTolerance; } set { _upsampleTolerance = value; } }

        [SerializeField, Range(1, 10)] float _thicknessModifier = 1;
        public float thicknessModifier { get { return _thicknessModifier; } set { _thicknessModifier = value; } }

        [SerializeField, Range(0, 2)] float _intensity = 1;
        public float intensity { get { return _intensity; } set { _intensity = value; } }

        [SerializeField, Range(0, 17)] int _debug;

        [SerializeField] bool _ambientOnly = true;
        public bool ambientOnly { get { return _ambientOnly; } set { _ambientOnly = value; } }

        // ---- not in the reference inspector: the shader variants Render.compute / Upsample.compute ship but AO.cs never selects ----
        [SerializeField] bool _sampleExhaustively;             // Render.compute:144-159, AmbientOcclusion.cs:709-715 (FIXME there)
        [SerializeField, Range(0, 15)] int _highQualityMask;   // bit k-1: Render kernel "main" on level k + Upsample "main_premin*"
        // Layered frames (meao_set_layers): views per frame, rendered together -- 2 for the eye slices of a texture-array (instanced)
        // stereo target, 6 for cube-map faces.  The depth and AO buffers the interop layer maps then hold Layers images each.
        [SerializeField, Range(1, 65535)] int _layers = 1;
        public int Layers { get { return _layers; } set { _layers = value; } }
        // One camera per layer (split-screen viewports, mirrors and portals, frames of several cameras in one batch); null: every layer
        // renders with this component's camera.  Each must have this camera's pixel size; Length must equal Layers.
        Camera[] _layerCameras;
        public Camera[] LayerCameras { get { return _layerCameras; } set { _layerCameras = value; } }
        // Dynamic resolution scaling: the largest camera pixel size the render size moves within (zero: none).  Reserved once
        // (meao_reserve); a size change inside it then costs no allocation, device synchronise, graph teardown or event rebind.
        Vector2Int _maxResolution;
        public Vector2Int MaxResolution { get { return _maxResolution; } set { _maxResolution = value; } }
        int _reservedW, _reservedH;                            // what meao_reserve was last given (doubled width under single-pass stereo)
        int _width, _height;                                   // the size meao_resize was last given
        int _drawCountPerFrame;                                // AmbientOcclusion.cs:289, 349-355: single-pass stereo detection
        void OnPreRender() { _drawCountPerFrame++; }
        bool singlePassStereoEnabled                           // AmbientOcclusion.cs:392-401
        {
            get { return _camera != null && _camera.stereoEnabled && _camera.targetTexture == null && _drawCountPerFrame == 1; }
        }

        const int kEventId = 0x4d41;   // "MA"

        Camera _camera;
        IntPtr _ctx = IntPtr.Zero;
        CommandBuffer _renderCommand;
        IntPtr _depthDev = IntPtr.Zero, _aoDev = IntPtr.Zero;   // mapped by the engine-specific interop layer
        // ... or, when the interop layer maps the textures as CUDA arrays (cudaArray_t of the depth copy and the R8 AO target,
        // registered with cudaGraphicsRegisterFlagsSurfaceLoadStore), those: the plugin event then reads and writes them directly
        IntPtr _depthArray = IntPtr.Zero, _aoArray = IntPtr.Zero;
        int _depthArrayKind = 0;                                // MEAO_DEPTH_RAW_F32 (R32_FLOAT copy) or 2 = RAW_D16_UNORM (R16 copy)
        // ... or, when the interop layer maps linear buffers that keep the graphics API's row pitch (a D3D12 footprint rounds each row up
        // to 256 bytes; a dynamic-resolution frame is the corner of a max-size target), their byte pitches; 0 = tight (meao_bind_event)
        long _depthRowPitch, _depthLayerPitch, _aoRowPitch, _aoLayerPitch;
        IntPtr _stream = IntPtr.Zero;                           // cudaStream_t the plugin event renders on (ABI 3; Zero = legacy default stream)

        void LateUpdate()
        {
            if (_camera == null)
            {
                _camera = GetComponent<Camera>();
                _camera.depthTextureMode = DepthTextureMode.Depth;          // AmbientOcclusion.cs:447
            }
            if (_ctx == IntPtr.Zero)
            {
                var cfg = new MeaoNative.MeaoDeviceCfg { device = 0, flags = 0 };
                MeaoNative.Check(IntPtr.Zero, MeaoNative.meao_create(ref cfg, out _ctx));
            }

            // CheckPropertiesChanged + CheckBaseDimensions live inside the plugin: the setters return 1
            // when the plan was dirtied (AmbientOcclusion.cs:104-113, 338-341).
            var p = new MeaoNative.MeaoParams
            {
                noise_filter_tolerance = _noiseFilterTolerance, blur_tolerance = _blurTolerance,
                upsample_tolerance = _upsampleTolerance, thickness_modifier = _thicknessModifier,
                intensity = _intensity, debug = _debug, ambient_only = _ambientOnly ? 1 : 0
            };
            var rebuild = MeaoNative.meao_set_params(_ctx, ref p) == 1;

            var cam = new MeaoNative.MeaoCamera
            {
                near_clip = _camera.nearClipPlane, far_clip = _camera.farClipPlane,          // :563
                tan_half_fov_h = 1 / _camera.projectionMatrix[0, 0],                         // :570-573
                reversed_z = SystemInfo.usesReversedZBuffer ? 1 : 0                          // :564
            };
            MeaoNative.Check(_ctx, MeaoNative.meao_set_camera(_ctx, ref cam));
            var stereo = singlePassStereoEnabled;
            var variants = new MeaoNative.MeaoVariants
            {
                single_pass_stereo = stereo ? 1 : 0,                                         // :680
                sample_exhaustively = _sampleExhaustively ? 1 : 0, high_quality_mask = _highQualityMask,
                single_scale = 0                                                             // BASELINE configs[0] plumbing mode; the component never selects it
            };
            rebuild |= MeaoNative.meao_set_variants(_ctx, ref variants) == 1;
            var layered = MeaoNative.meao_set_layers(_ctx, _layers);
            MeaoNative.Check(_ctx, layered);
            rebuild |= layered == 1;
            rebuild |= SetLayerCameras() == 1;                                               // after meao_set_layers, which clears the table
            var width = _camera.pixelWidth * (stereo ? 2 : 1);
            rebuild |= Reserve(width, _camera.pixelHeight, stereo);                          // before meao_resize, doubled like the width
            var resized = MeaoNative.meao_resize(_ctx, width, _camera.pixelHeight);          // :338-341
            MeaoNative.Check(_ctx, resized);
            rebuild |= resized == 1 && _reservedW == 0;     // inside a reservation the bound event renders the new size as it is
            _width = width; _height = _camera.pixelHeight;
            rebuild |= !Application.isPlaying;                                               // :345
            _drawCountPerFrame = 0;                                                          // :349

            if (rebuild || _renderCommand == null) RebuildCommandBuffers();
        }

        // Hands MaxResolution to meao_reserve; true if the arena was re-allocated.  When the current size does not fit the new
        // reservation, the context first drops its reservation and takes the new size (meao_reserve refuses a reservation below it).
        bool Reserve(int width, int height, bool stereo)
        {
            int w = _maxResolution.x * (stereo ? 2 : 1), h = _maxResolution.y;
            if (_maxResolution.x <= 0 || _maxResolution.y <= 0) w = h = 0;
            if (w == _reservedW && h == _reservedH) return false;
            if (w != 0 && (_width > w || _height > h))
            {
                MeaoNative.Check(_ctx, MeaoNative.meao_reserve(_ctx, 0, 0));
                _reservedW = _reservedH = 0;
                MeaoNative.Check(_ctx, MeaoNative.meao_resize(_ctx, width, height));
            }
            MeaoNative.Check(_ctx, MeaoNative.meao_reserve(_ctx, w, h));
            _reservedW = w; _reservedH = h;
            return true;
        }

        // Hands LayerCameras to the plugin; returns 1 if it re-planned.  The same table again returns 0, so this runs every frame.
        int SetLayerCameras()
        {
            if (_layerCameras == null) return MeaoNative.meao_set_layer_cameras(_ctx, null, 0);
            var cams = new MeaoNative.MeaoCamera[_layerCameras.Length];
            for (int i = 0; i < cams.Length; i++)
            {
                var c = _layerCameras[i];
                if (c.pixelWidth != _camera.pixelWidth || c.pixelHeight != _camera.pixelHeight)
                    throw new ArgumentException("LayerCameras[" + i + "] has another pixel size than the camera");
                cams[i] = new MeaoNative.MeaoCamera
                {
                    near_clip = c.nearClipPlane, far_clip = c.farClipPlane,
                    tan_half_fov_h = 1 / c.projectionMatrix[0, 0],
                    reversed_z = SystemInfo.usesReversedZBuffer ? 1 : 0
                };
            }
            var rc = MeaoNative.meao_set_layer_cameras(_ctx, cams, cams.Length);
            MeaoNative.Check(_ctx, rc);
            return rc;
        }

        void RebuildCommandBuffers()
        {
            if (_renderCommand == null) _renderCommand = new CommandBuffer { name = "SSAO" };   // :481-482
            else _camera.RemoveCommandBuffer(CameraEvent.BeforeImageEffects, _renderCommand);
            _renderCommand.Clear();
            // (engine-specific: map _CameraDepthTexture and the R8 AO render texture to _depthDev / _aoDev, or to _depthArray / _aoArray)
            if (_depthArray != IntPtr.Zero) BindEventArrays();
            else if (_depthRowPitch != 0) BindEventPitched();
            else MeaoNative.Check(_ctx, MeaoNative.meao_bind_event(_ctx, kEventId, _depthDev, 0 /* MEAO_DEPTH_RAW_F32 */, _aoDev, _stream));
            // one plugin event replaces the ten DispatchCompute calls recorded by :511-531
            _renderCommand.IssuePluginEvent(MeaoNative.meao_get_render_event_func(), kEventId);
            _camera.AddCommandBuffer(CameraEvent.BeforeImageEffects, _renderCommand);          // :421
        }

        // The array path of the plugin event: meao_render_arrays on the mapped arrays (checked here -- the event cannot report errors).
        void BindEventArrays()
        {
            MeaoNative.Check(_ctx, MeaoNative.meao_bind_event_arrays(_ctx, kEventId, _depthArray, _depthArrayKind, _aoArray, _stream));
        }

        // The pitched path of the plugin event: meao_render_pitched on the mapped buffers at their own pitches (checked here -- the
        // event cannot report errors).  With one layer the layer pitches are not used.
        void BindEventPitched()
        {
            MeaoNative.Check(_ctx, MeaoNative.meao_bind_event_pitched(_ctx, kEventId, _depthDev, _depthRowPitch, _depthLayerPitch, 0 /* MEAO_DEPTH_RAW_F32 */,
                                                                     _aoDev, _aoRowPitch, _aoLayerPitch, _stream));
        }

        // The interop layer calls this before it unmaps, unregisters or re-creates a texture it handed over as an array: the plugin
        // caches a surface object and graphs per array, and a new array may come back with the same handle.
        public void ReleaseArrays()
        {
            if (_ctx == IntPtr.Zero) return;
            if (_depthArray != IntPtr.Zero) MeaoNative.Check(_ctx, MeaoNative.meao_release_array(_ctx, _depthArray));
            if (_aoArray != IntPtr.Zero) MeaoNative.Check(_ctx, MeaoNative.meao_release_array(_ctx, _aoArray));
            _depthArray = _aoArray = IntPtr.Zero;
        }

        void OnDisable()
        {
            if (_renderCommand != null && _camera != null)
                _camera.RemoveCommandBuffer(CameraEvent.BeforeImageEffects, _renderCommand);
        }

        void OnDestroy()
        {
            if (_ctx != IntPtr.Zero) { MeaoNative.meao_destroy(_ctx); _ctx = IntPtr.Zero; }    // :357-381
            if (_renderCommand != null) { _renderCommand.Dispose(); _renderCommand = null; }
        }
    }
}
