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

        // Where layer l of a CUDA-array frame reads its depth and writes its AO (meao.h: MeaoLayerViewport)
        [StructLayout(LayoutKind.Sequential)]
        public struct MeaoLayerViewport
        {
            public int depth_x, depth_y, depth_slice;
            public int ao_x, ao_y, ao_slice;
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
        [DllImport(Lib)] public static extern int meao_set_hierarchy_depth(IntPtr ctx, int levels);
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
        // lay the intermediates out once for the most layers; a layer change up to it then allocates and synchronises nothing (0 clears)
        [DllImport(Lib)] public static extern int meao_reserve_layers(IntPtr ctx, int maxLayers);
        [DllImport(Lib)] public static extern int meao_layer_reservation(IntPtr ctx);
        // one camera per layer (split-screen viewports, mirrors, batches from several cameras); null with count 0 clears the table
        [DllImport(Lib)] public static extern int meao_set_layer_cameras(IntPtr ctx, [In] MeaoCamera[] cameras, int count);
        [DllImport(Lib)] public static extern int meao_get_layer_cameras(IntPtr ctx, [Out] MeaoCamera[] cameras, int capacity);
        [DllImport(Lib)] public static extern int meao_set_layer_viewports(IntPtr ctx, [In] MeaoLayerViewport[] views, int count);
        [DllImport(Lib)] public static extern int meao_get_layer_viewports(IntPtr ctx, [Out] MeaoLayerViewport[] views, int capacity);
        [DllImport(Lib)] public static extern int meao_render(IntPtr ctx, IntPtr depthDev, int depthKind, IntPtr aoOutDev, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_render_host(IntPtr ctx, float[] depth, int depthKind, byte[] aoOut);
        [DllImport(Lib)] public static extern int meao_bind_event(IntPtr ctx, int eventId, IntPtr depthDev, int depthKind, IntPtr aoOutDev, IntPtr stream);
        // CUDA arrays (graphics interop: cudaGraphicsSubResourceGetMappedArray / level 0 of a Vulkan mipmapped array), no copies
        [DllImport(Lib)] public static extern int meao_render_arrays(IntPtr ctx, IntPtr depthArray, int depthKind, IntPtr aoArray, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_bind_event_arrays(IntPtr ctx, int eventId, IntPtr depthArray, int depthKind, IntPtr aoArray, IntPtr stream);
        // ... or a viewport of larger arrays: the frame's W x H texels at (depthX, depthY) and (aoX, aoY) -- max-size targets of a
        // dynamic-resolution engine, one player's half of a split-screen texture
        [DllImport(Lib)] public static extern int meao_render_arrays_at(IntPtr ctx, IntPtr depthArray, int depthX, int depthY, int depthKind,
                                                                        IntPtr aoArray, int aoX, int aoY, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_bind_event_arrays_at(IntPtr ctx, int eventId, IntPtr depthArray, int depthX, int depthY, int depthKind,
                                                                            IntPtr aoArray, int aoX, int aoY, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_release_array(IntPtr ctx, IntPtr array);   // before the array is unmapped / unregistered / freed
        // Batches: layer l of a layered frame reads depthArrays[l] and writes aoArrays[l] -- several cameras, each with its own targets
        // (count = meao_set_layers, at most MEAO_MAX_BATCH = 256; each array 2-D, at least W x H, the frame at its top-left corner)
        [DllImport(Lib)] public static extern int meao_render_arrays_batch(IntPtr ctx, [In] IntPtr[] depthArrays, int depthKind, [In] IntPtr[] aoArrays,
                                                                           int count, IntPtr stream);
        [DllImport(Lib)] public static extern int meao_bind_event_arrays_batch(IntPtr ctx, int eventId, [In] IntPtr[] depthArrays, int depthKind,
                                                                               [In] IntPtr[] aoArrays, int count, IntPtr stream);
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
        // frames recorded into the host's own CUDA graph (a render called on a capturing stream) replay only while this is unchanged
        [DllImport(Lib)] public static extern long meao_frame_generation(IntPtr ctx);
        // MEAO_PROJECTION_PERSPECTIVE 0 / MEAO_PROJECTION_ORTHOGRAPHIC 1 (Camera.orthographic): a structural input, one per context.  Under
        // an orthographic camera 1 / projectionMatrix[0,0] is the view volume's half-width, and LINEAR_F32 depth must be eye depth / far
        [DllImport(Lib)] public static extern int meao_set_projection(IntPtr ctx, int projection);
        [DllImport(Lib)] public static extern int meao_get_projection(IntPtr ctx);
        // one projection per layer (an editor's quad view, a bird's-eye-view camera beside perspective sensors): count = meao_set_layers,
        // null with count 0 clears the table, which then decides each layer's projection alone (a structural input)
        [DllImport(Lib)] public static extern int meao_set_layer_projections(IntPtr ctx, [In] int[] projections, int count);
        [DllImport(Lib)] public static extern int meao_get_layer_projections(IntPtr ctx, [Out] int[] projections, int capacity);
        // Cameras read from device memory at every launch and graph replay (meao_bind_device_cameras).  Declarations only: a Unity host has
        // no CUDA buffer of its own to hand over; a native plugin or an interop host that keeps its cameras on the GPU passes its pointer.
        [DllImport(Lib)] public static extern int meao_bind_device_cameras(IntPtr ctx, IntPtr camerasDev, int capacity);
        [DllImport(Lib)] public static extern int meao_device_camera_status(IntPtr ctx, [Out] int[] out4);
        // Thickness modifier and intensity read from device memory at every launch and graph replay (meao_bind_device_params).
        // Declarations only, like the device cameras: a native plugin or an interop host that animates them on the GPU passes its pointer.
        [DllImport(Lib)] public static extern int meao_bind_device_params(IntPtr ctx, IntPtr paramsDev);
        [DllImport(Lib)] public static extern int meao_device_param_status(IntPtr ctx, [Out] int[] out4);

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
        // The levels of the AO pyramid a frame renders and upsamples (upstream MiniEngine's "Hierarchy Depth"): 4 is the reference's
        // frame; fewer cost less and drop the coarsest, large-scale darkening.  A change re-plans the plugin (a device synchronise).
        [SerializeField, Range(1, 4)] int _hierarchyDepth = 4;
        public int HierarchyDepth { get { return _hierarchyDepth; } set { _hierarchyDepth = value; } }
        // Layered frames (meao_set_layers): views per frame, rendered together -- 2 for the eye slices of a texture-array (instanced)
        // stereo target, 6 for cube-map faces.  The depth and AO buffers the interop layer maps then hold Layers images each.
        [SerializeField, Range(1, 65535)] int _layers = 1;
        public int Layers { get { return _layers; } set { _layers = value; } }
        // One camera per layer (split-screen viewports, mirrors and portals, frames of several cameras in one batch); null: every layer
        // renders with this component's camera.  Each must have this camera's pixel size; Length must equal Layers.
        Camera[] _layerCameras;
        public Camera[] LayerCameras { get { return _layerCameras; } set { _layerCameras = value; } }
        // Perspective and orthographic layers in one frame: true hands each LayerCameras[i].orthographic to the plugin as that layer's
        // projection (meao_set_layer_projections) instead of requiring it to match this camera's.
        bool _perLayerProjection;
        public bool PerLayerProjection { get { return _perLayerProjection; } set { _perLayerProjection = value; } }
        // Where each layer lives in the depth and AO targets (split-screen players in one texture, a side-by-side stereo pair, cube faces
        // in a 2-D atlas); null: every layer at the origin of its own slice.  Length must equal Layers.  Honoured by the frames of
        // meao_render, meao_render_pitched and meao_render_arrays and the events bound to them; the host-buffer calls, the stage calls,
        // the debug views and the composites keep the tight layer layout.
        MeaoNative.MeaoLayerViewport[] _layerViewports;
        public MeaoNative.MeaoLayerViewport[] LayerViewports { get { return _layerViewports; } set { _layerViewports = value; } }
        // Dynamic resolution scaling: the largest camera pixel size the render size moves within (zero: none).  Reserved once
        // (meao_reserve); a size change inside it then costs no allocation, device synchronise, graph teardown or event rebind.
        Vector2Int _maxResolution;
        public Vector2Int MaxResolution { get { return _maxResolution; } set { _maxResolution = value; } }
        // Dynamic view counts (split-screen players joining and leaving, visible cube faces): the most Layers the component will have
        // (zero: none).  Reserved once (meao_reserve_layers); a change of Layers up to it then costs no allocation, device synchronise
        // or graph teardown.
        int _maxLayers;
        public int MaxLayers { get { return _maxLayers; } set { _maxLayers = value; } }
        int _reservedLayers, _contextLayers = 1;               // what meao_reserve_layers / meao_set_layers were last given
        // An engine that records the plugin's frame into a CUDA graph of its own (meao_render on a stream it captures) replays that
        // graph only while this equals the value read right after the capture, and captures again when it changes (include/meao.h).
        public long FrameGeneration { get { return _ctx == IntPtr.Zero ? -1 : MeaoNative.meao_frame_generation(_ctx); } }
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
        // viewport origins in the arrays (BindEventArraysAt); null: the arrays are exactly the frame's size (meao_bind_event_arrays)
        Vector2Int? _depthArrayOrigin, _aoArrayOrigin;
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
            // the projection excludes a layer-viewport table: back to perspective before a table is set, orthographic after it is cleared
            if (!_camera.orthographic) rebuild |= SetProjection(0) == 1;
            var stereo = singlePassStereoEnabled;
            var variants = new MeaoNative.MeaoVariants
            {
                single_pass_stereo = stereo ? 1 : 0,                                         // :680
                sample_exhaustively = _sampleExhaustively ? 1 : 0, high_quality_mask = _highQualityMask,
                single_scale = 0                                                             // BASELINE configs[0] plumbing mode; the component never selects it
            };
            rebuild |= MeaoNative.meao_set_variants(_ctx, ref variants) == 1;
            var depthChanged = MeaoNative.meao_set_hierarchy_depth(_ctx, _hierarchyDepth);              // a structural input, like the variants
            MeaoNative.Check(_ctx, depthChanged);
            rebuild |= depthChanged == 1;
            rebuild |= ReserveLayers();                                                      // before meao_set_layers
            var layered = SetLayers(_layers);
            rebuild |= layered == 1;
            rebuild |= SetLayerCameras() == 1;                                               // after meao_set_layers, which clears the table
            // an orthographic layer excludes a layer-viewport table: the projection table is cleared before the viewports and set after them
            var perLayer = _perLayerProjection && _layerCameras != null;
            if (!perLayer) rebuild |= SetLayerProjections(false) == 1;
            var viewports = _layerViewports == null ? MeaoNative.meao_set_layer_viewports(_ctx, null, 0)
                                                    : MeaoNative.meao_set_layer_viewports(_ctx, _layerViewports, _layerViewports.Length);
            MeaoNative.Check(_ctx, viewports);
            rebuild |= viewports == 1;                                                       // after meao_set_layers too
            if (perLayer) rebuild |= SetLayerProjections(true) == 1;
            if (_camera.orthographic) rebuild |= SetProjection(1) == 1;
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

        int SetLayers(int layers)
        {
            var rc = MeaoNative.meao_set_layers(_ctx, layers);
            MeaoNative.Check(_ctx, rc);
            _contextLayers = layers;
            return rc;
        }

        // Hands MaxLayers to meao_reserve_layers; true if the arena was re-allocated.  When the context has more layers than the new
        // reservation, it first takes Layers (meao_reserve_layers refuses a reservation below the current count).
        bool ReserveLayers()
        {
            var want = _maxLayers > 0 ? _maxLayers : 0;
            if (want != 0 && _layers > want) throw new InvalidOperationException("Layers " + _layers + " lies above MaxLayers " + want);
            if (want == _reservedLayers) return false;
            if (want != 0 && _contextLayers > want) SetLayers(_layers);
            MeaoNative.Check(_ctx, MeaoNative.meao_reserve_layers(_ctx, want));
            _reservedLayers = want;
            return true;
        }

        // Hands the projection to the plugin (0 perspective, 1 orthographic); returns 1 if it changed (a re-plan), 0 if not.
        int SetProjection(int projection)
        {
            var rc = MeaoNative.meao_set_projection(_ctx, projection);
            MeaoNative.Check(_ctx, rc);
            return rc;
        }

        // Hands LayerCameras to the plugin; returns 1 if a value changed (the next frame takes it without a re-plan).  The same table again returns 0, so this runs every frame.
        int SetLayerCameras()
        {
            if (_layerCameras == null) return MeaoNative.meao_set_layer_cameras(_ctx, null, 0);
            var cams = new MeaoNative.MeaoCamera[_layerCameras.Length];
            for (int i = 0; i < cams.Length; i++)
            {
                var c = _layerCameras[i];
                if (c.pixelWidth != _camera.pixelWidth || c.pixelHeight != _camera.pixelHeight)
                    throw new ArgumentException("LayerCameras[" + i + "] has another pixel size than the camera");
                if (!_perLayerProjection && c.orthographic != _camera.orthographic)
                    throw new ArgumentException("LayerCameras[" + i + "] has another projection than the camera (set PerLayerProjection to mix them)");
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

        // Hands the projections of LayerCameras to the plugin (set), or clears the table (!set); returns 1 if it changed (a re-plan), 0 if
        // not, so this runs every frame.
        int SetLayerProjections(bool set)
        {
            int rc;
            if (!set) rc = MeaoNative.meao_set_layer_projections(_ctx, null, 0);
            else
            {
                var projections = new int[_layerCameras.Length];
                for (int i = 0; i < projections.Length; i++) projections[i] = _layerCameras[i].orthographic ? 1 : 0;
                rc = MeaoNative.meao_set_layer_projections(_ctx, projections, projections.Length);
            }
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

        // The array path of the plugin event: meao_render_arrays on the mapped arrays (checked here -- the event cannot report errors),
        // or meao_render_arrays_at at the origins BindEventArraysAt set.
        void BindEventArrays()
        {
            if (_depthArrayOrigin == null && _aoArrayOrigin == null)
            {
                MeaoNative.Check(_ctx, MeaoNative.meao_bind_event_arrays(_ctx, kEventId, _depthArray, _depthArrayKind, _aoArray, _stream));
                return;
            }
            Vector2Int d = _depthArrayOrigin ?? Vector2Int.zero, a = _aoArrayOrigin ?? Vector2Int.zero;
            MeaoNative.Check(_ctx, MeaoNative.meao_bind_event_arrays_at(_ctx, kEventId, _depthArray, d.x, d.y, _depthArrayKind, _aoArray, a.x, a.y, _stream));
        }

        // Dynamic resolution or split-screen on interop textures: the plugin event renders the frame's current W x H from the depth
        // array's texels at depthOrigin into the AO array's at aoOrigin.  Register and map the textures once at their largest size and
        // bind once: the event checks the viewport again at each frame's size, so a MaxResolution reservation needs no rebinding.
        public void BindEventArraysAt(IntPtr depthArray, Vector2Int depthOrigin, IntPtr aoArray, Vector2Int aoOrigin, int depthKind = 0)
        {
            _depthArray = depthArray; _aoArray = aoArray; _depthArrayKind = depthKind;
            _depthArrayOrigin = depthOrigin; _aoArrayOrigin = aoOrigin;
            if (_ctx != IntPtr.Zero) BindEventArrays();
        }

        // One frame from and into viewports of the arrays, outside the command buffer (a second camera's half of a split-screen target).
        public void RenderArraysAt(IntPtr depthArray, Vector2Int depthOrigin, IntPtr aoArray, Vector2Int aoOrigin, int depthKind = 0)
        {
            MeaoNative.Check(_ctx, MeaoNative.meao_render_arrays_at(_ctx, depthArray, depthOrigin.x, depthOrigin.y, depthKind, aoArray,
                                                                    aoOrigin.x, aoOrigin.y, _stream));
        }

        // One frame of every camera of a batch, each layer from and into its own mapped arrays (meao_render_arrays_batch): the
        // context's layer count must equal the list length.  Release each array with meao_release_array before it is unmapped.
        public void RenderArraysBatch(IntPtr[] depthArrays, IntPtr[] aoArrays, int depthKind = 0)
        {
            if (depthArrays.Length != aoArrays.Length) throw new ArgumentException("one depth and one AO array per layer");
            MeaoNative.Check(_ctx, MeaoNative.meao_render_arrays_batch(_ctx, depthArrays, depthKind, aoArrays, depthArrays.Length, _stream));
        }

        // The plugin event renders the batch: the library copies the lists and checks them now (the event cannot report errors).
        public void BindEventArraysBatch(IntPtr[] depthArrays, IntPtr[] aoArrays, int depthKind = 0)
        {
            if (depthArrays.Length != aoArrays.Length) throw new ArgumentException("one depth and one AO array per layer");
            MeaoNative.Check(_ctx, MeaoNative.meao_bind_event_arrays_batch(_ctx, kEventId, depthArrays, depthKind, aoArrays, depthArrays.Length,
                                                                           _stream));
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
            _depthArrayOrigin = _aoArrayOrigin = null;
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
