// depth_in.cuh -- reading and linearising the caller's raw depth (Downsample1.compute Linearize, DS1:37-48), shared by the two
// stages that read it: prepare_depth (prepare_depth_kernel.inc) and the final upsample of a whole frame (blur_upsample_lin.cu),
// which linearises its own pixels and writes LinearDepth itself.  Included inside an anonymous namespace.

#if MEAO_ORTHO == 2
// MEAO_ORTHO 2 (the *_mixed kernels, meao_set_layer_projections): both linearisations below, under the names of their projection; the
// linearize8 at the end picks one per call from a CTA-uniform flag
#define linearize linearize_persp
#define linearize8 linearize8_persp
#endif
#if MEAO_ORTHO != 1
template <bool RAW, bool REVERSED>
__device__ __forceinline__ float linearize(float depth, float zbx, float zby)
{
    if (!RAW) return depth;
    float dist = rcp_ieee(fmaf(zbx, depth, zby));       // DS1:40 (mad + IEEE reciprocal)
    if (REVERSED) { if (depth == 0.0f) dist = 1e5f; }   // DS1:41-42
    else          { if (depth == 1.0f) dist = 1e5f; }   // DS1:43-44
    return dist;
}

// Eight pixels at once: the mad of DS1:40 is formed directly in negated form, nt = fma(-zbx, d, -zby) = -t
// exactly (round-to-nearest is sign-symmetric), all eight range tests feed ONE branch, and the reciprocals run in pairs
// (rcp2_fast_neg).  If any element is out of range (inf / NaN / zero / denormal / negative) the group takes the plain
// per-element path of linearize() -- which recomputes t itself, so signed zeros behave exactly as before.
template <bool RAW, bool REVERSED>
__device__ __forceinline__ void linearize8(const float (&v)[8], float zbx, float zby, float (&d)[8])
{
    if (!RAW) {
#pragma unroll
        for (int e = 0; e < 8; e++) d[e] = v[e];
        return;
    }
    const float2 nzx = make_float2(-zbx, -zbx), nzy = make_float2(-zby, -zby);
    float2 nt[4];
    bool ok = true;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        nt[q] = ffma2(make_float2(v[2 * q], v[2 * q + 1]), nzx, nzy);
        ok = ok & in_safe_range_neg(nt[q].x) & in_safe_range_neg(nt[q].y);
    }
    if (ok) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const float2 r = rcp2_fast_neg(nt[q]);
            d[2 * q] = r.x; d[2 * q + 1] = r.y;
        }
#pragma unroll
        for (int e = 0; e < 8; e++) {
            if (REVERSED) { if (v[e] == 0.0f) d[e] = 1e5f; }   // DS1:41-42
            else          { if (v[e] == 1.0f) d[e] = 1e5f; }   // DS1:43-44
        }
    } else {
#pragma unroll
        for (int e = 0; e < 8; e++) d[e] = linearize<RAW, REVERSED>(v[e], zbx, zby);
    }
}
#endif
#if MEAO_ORTHO == 2
#undef linearize8
#undef linearize
#define linearize linearize_ortho
#define linearize8 linearize8_ortho
#endif
#if MEAO_ORTHO
// An orthographic projection (MEAO_ORTHO: the *_ortho kernels, meao_set_projection) stores depth that is affine in eye depth, so the
// linear depth is one fused multiply-add: zb = {1 - n/f, n/f} (reversed: {n/f - 1, 1}) gives eye depth / far, LinearDepth's
// convention.  The sky rule of DS1:41-44 is the perspective one.  No reciprocal, so no range test.
template <bool RAW, bool REVERSED>
__device__ __forceinline__ float linearize(float depth, float zbx, float zby)
{
    if (!RAW) return depth;
    float dist = fmaf(zbx, depth, zby);
    if (REVERSED) { if (depth == 0.0f) dist = 1e5f; }
    else          { if (depth == 1.0f) dist = 1e5f; }
    return dist;
}

template <bool RAW, bool REVERSED>
__device__ __forceinline__ void linearize8(const float (&v)[8], float zbx, float zby, float (&d)[8])
{
    if (!RAW) {
#pragma unroll
        for (int e = 0; e < 8; e++) d[e] = v[e];
        return;
    }
    const float2 zx = make_float2(zbx, zbx), zy = make_float2(zby, zby);
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const float2 r = ffma2(make_float2(v[2 * q], v[2 * q + 1]), zx, zy);
        d[2 * q] = r.x; d[2 * q + 1] = r.y;
    }
#pragma unroll
    for (int e = 0; e < 8; e++) {
        if (REVERSED) { if (v[e] == 0.0f) d[e] = 1e5f; }
        else          { if (v[e] == 1.0f) d[e] = 1e5f; }
    }
}
#endif
#if MEAO_ORTHO == 2
#undef linearize8
#undef linearize
// A layer's linearisation by its projection: `ortho` is uniform across the CTA (one layer's, read once), so each call runs one of the
// two loops above as its twin kernel does
template <bool RAW, bool REVERSED>
__device__ __forceinline__ void linearize8(const float (&v)[8], float zbx, float zby, float (&d)[8], bool ortho)
{
    if (ortho) linearize8_ortho<RAW, REVERSED>(v, zbx, zby, d);
    else linearize8_persp<RAW, REVERSED>(v, zbx, zby, d);
}
#endif

// native depth formats (SURVEY.md 8f.1): the camera depth texture read by Blit.shader pass 0 (:48-64) is a D32_FLOAT,
// D24_UNORM_S8_UINT or D16_UNORM resource; SAMPLE_DEPTH_TEXTURE returns code / (2^n - 1) for the UNORM ones
// (D3D UNORM -> FLOAT rule: (float)code * (1.0f / (2^n - 1))).
enum { IN_F32 = 0, IN_D16 = 1, IN_D24S8 = 2 };

template <int IN>
__device__ __forceinline__ void load8(const void *base, size_t elem_index, bool full, int valid, float (&v)[8])
{
    if (IN == IN_F32) {
        const float *src = reinterpret_cast<const float *>(base) + elem_index;
        if (full) {
            const float4 q0 = ldg_stream_f4(src), q1 = ldg_stream_f4(src + 4);
            v[0] = q0.x; v[1] = q0.y; v[2] = q0.z; v[3] = q0.w; v[4] = q1.x; v[5] = q1.y; v[6] = q1.z; v[7] = q1.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; e++) v[e] = (e < valid) ? __ldg(src + e) : 0.0f;
        }
    } else if (IN == IN_D16) {
        const uint16_t *src = reinterpret_cast<const uint16_t *>(base) + elem_index;
        uint32_t c[8];
        if (full) {
            const uint4 q = ldg_stream_u4(src);
            c[0] = q.x & 0xffffu; c[1] = q.x >> 16; c[2] = q.y & 0xffffu; c[3] = q.y >> 16;
            c[4] = q.z & 0xffffu; c[5] = q.z >> 16; c[6] = q.w & 0xffffu; c[7] = q.w >> 16;
        } else {
#pragma unroll
            for (int e = 0; e < 8; e++) c[e] = (e < valid) ? __ldg(src + e) : 0u;
        }
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = __fmul_rn((float)c[e], 1.0f / 65535.0f);
    } else {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(base) + elem_index;
        uint32_t c[8];
        if (full) {
            const uint4 q0 = ldg_stream_u4(src), q1 = ldg_stream_u4(src + 4);
            c[0] = q0.x; c[1] = q0.y; c[2] = q0.z; c[3] = q0.w; c[4] = q1.x; c[5] = q1.y; c[6] = q1.z; c[7] = q1.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; e++) c[e] = (e < valid) ? __ldg(src + e) : 0u;
        }
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = __fmul_rn((float)(c[e] & 0xffffffu), 1.0f / 16777215.0f);   // depth = low 24 bits, stencil = high 8
    }
}
