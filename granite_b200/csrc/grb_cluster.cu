// grb_cluster.cu -- the bindless light clusterer (spot hull transform, per-light cull setup,
// XY tile binning, per-slice Z range) as sm_90a kernels.  Compiled with -fmad=false: the
// outputs are integers (bitmask words, index ranges) decided by fp32 comparisons, and the
// contract with the reference/oracle is bit-exactness, so every fp32 op must round on its own.
//
// Replaces LightClusterer::build_cluster_bindless_gpu (renderer/lights/clusterer.cpp:1463-1573).
#include "grb_common.cuh"

#include <cstdlib>

namespace grb
{
namespace
{
struct CamDev
{
	float view[16];
	float vp[16];
	float3 pos, front;
	float z_near, z_far;
};

__device__ __forceinline__ float4 mul_m4(const float *m, float x, float y, float z, float w)
{
	return make_float4(m[0] * x + m[4] * y + m[8] * z + m[12] * w, m[1] * x + m[5] * y + m[9] * z + m[13] * w,
	                   m[2] * x + m[6] * y + m[10] * z + m[14] * w, m[3] * x + m[7] * y + m[11] * z + m[15] * w);
}

__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float3 add3(float3 a, float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 sub3(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float len2(float x, float y) { return sqrtf(x * x + y * y); }

// ------------------------------------------------------------------------------- K1
// One thread per light: 5 cone-hull points -> clip space, view-Z extent, cull sign.
__global__ void __launch_bounds__(128) spot_transform_kernel(CamDev cam, const float *__restrict__ model, int num_lights, float4 *__restrict__ out)
{
	int index = blockIdx.x * blockDim.x + threadIdx.x;
	if (index >= num_lights)
		return;
	const float4 *m = reinterpret_cast<const float4 *>(model) + (size_t)index * 3;
	float4 r0 = __ldg(m), r1 = __ldg(m + 1), r2 = __ldg(m + 2);
	float3 p[5];
	p[0] = make_float3(r0.w, r1.w, r2.w);
	float3 pz = add3(p[0], make_float3(-r0.z, -r1.z, -r2.z));
	float3 right = make_float3(r0.x, r1.x, r2.x);
	float3 up = make_float3(r0.y, r1.y, r2.y);
	p[1] = add3(add3(pz, right), up);
	p[2] = add3(sub3(pz, right), up);
	p[3] = sub3(sub3(pz, right), up);
	p[4] = sub3(add3(pz, right), up);
	float z_lo = 0.0f, z_hi = 0.0f;
#pragma unroll
	for (int i = 0; i < 5; i++)
	{
		float z = dot3(sub3(p[i], cam.pos), cam.front);
		z_lo = i == 0 ? z : fmin_(z_lo, z);
		z_hi = i == 0 ? z : fmax_(z_hi, z);
	}
	float cull;
	if (z_lo <= cam.z_near && z_hi >= cam.z_far)
		cull = 0.0f;
	else if (z_lo <= cam.z_near)
		cull = -1.0f;
	else
		cull = 1.0f;
	float4 *o = out + (size_t)index * 6;
#pragma unroll
	for (int i = 0; i < 5; i++)
		o[i] = mul_m4(cam.vp, p[i].x, p[i].y, p[i].z, 1.0f);
	o[5] = make_float4(cull, z_lo, z_hi, 0.0f);
}

// ------------------------------------------------------------------------------- K2
__device__ __forceinline__ float2 project_sphere_flat(float view_xy, float view_z, float radius)
{
	float len = len2(view_xy, view_z);
	float sin_xy = radius / len;
	if (sin_xy < 0.999f)
	{
		float cos_xy = sqrtf(1.0f - sin_xy * sin_xy);
		float2 rot_lo = make_float2(cos_xy * view_xy + (-sin_xy) * view_z, sin_xy * view_xy + cos_xy * view_z);
		float2 rot_hi = make_float2(cos_xy * view_xy + sin_xy * view_z, (-sin_xy) * view_xy + cos_xy * view_z);
		if (rot_lo.y <= 0.0f)
			rot_lo = make_float2(-1.0f, 0.0f);
		if (rot_hi.y <= 0.0f)
			rot_hi = make_float2(+1.0f, 0.0f);
		return make_float2(rot_lo.x / rot_lo.y, rot_hi.x / rot_hi.y);
	}
	return make_float2(-INFINITY, +INFINITY);
}

struct Tri2 { float2 c[3]; };
struct Tri3 { float3 c[3]; };

__device__ __forceinline__ float3 mix3(float3 a, float3 b, float t)
{
	float it = 1.0f - t;
	return make_float3(a.x * it + b.x * t, a.y * it + b.y * t, a.z * it + b.z * t);
}

__device__ __forceinline__ float4 mix4(float4 a, float4 b, float t)
{
	float it = 1.0f - t;
	return make_float4(a.x * it + b.x * t, a.y * it + b.y * t, a.z * it + b.z * t, a.w * it + b.w * t);
}

__device__ __forceinline__ float3 xyz_div(float4 c, float d) { return make_float3(c.x / d, c.y / d, c.z / d); }
__device__ __forceinline__ float cross2(float2 a, float2 b) { return a.x * b.y - a.y * b.x; }
__device__ __forceinline__ float sign1(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }

constexpr uint32_t kMaxTriangles = 8u;

__device__ void emit_triangle(uint32_t &count, const Tri2 &t, float cull, float4 *data)
{
	float2 c0 = t.c[0], c1 = t.c[1], c2 = t.c[2];
	float2 ab = make_float2(c1.x - c0.x, c1.y - c0.y);
	float2 bc = make_float2(c2.x - c1.x, c2.y - c1.y);
	float2 ca = make_float2(c0.x - c2.x, c0.y - c2.y);
	float z = cross2(ab, make_float2(-ca.x, -ca.y));
	if (fabsf(z) < 0.000001f || sign1(cull) == sign1(z))
		return;
	float inv_z = 1.0f / z;
	if (count < kMaxTriangles)
	{
		float4 *d = data + 4u * count;
		d[0] = make_float4(inv_z * cross2(ab, make_float2(-c0.x, -c0.y)), inv_z * cross2(bc, make_float2(-c1.x, -c1.y)),
		                   inv_z * cross2(ca, make_float2(-c2.x, -c2.y)), 0.0f);
		d[1] = make_float4(inv_z * -ab.y, inv_z * -bc.y, inv_z * -ca.y, z);
		d[2] = make_float4(inv_z * ab.x, inv_z * bc.x, inv_z * ca.x, inv_z);
		d[3] = make_float4(fmin_(fmin_(c0.x, c1.x), c2.x), fmin_(fmin_(c0.y, c1.y), c2.y), fmax_(fmax_(c0.x, c1.x), c2.x),
		                   fmax_(fmax_(c0.y, c1.y), c2.y));
	}
	count++;
}

// clip a projected triangle against z < 0 (far side of reverse-Z clip space)
__device__ void clip_z_and_emit(uint32_t &count, const Tri3 &t, float cull, float4 *data)
{
	float3 c[3] = { t.c[0], t.c[1], t.c[2] };
	uint32_t code = (uint32_t)(c[0].z < 0.0f) + (uint32_t)(c[1].z < 0.0f) * 2u + (uint32_t)(c[2].z < 0.0f) * 4u;
	if (code == 7u)
		return;
	Tri2 k0, k1;
	bool dual = false;
	if (code == 0u)
	{
		k0.c[0] = make_float2(c[0].x, c[0].y);
		k0.c[1] = make_float2(c[1].x, c[1].y);
		k0.c[2] = make_float2(c[2].x, c[2].y);
	}
	else
	{
		// rotation so that the special vertex ordering of the reference's switch is reproduced:
		// one vertex out (codes 1,2,4): (out, next, next2); two out (3,5,6): (out_a, out_b, in)
		int r = (code == 1u || code == 3u) ? 0 : ((code == 2u || code == 6u) ? 1 : 2);
		float3 a = c[r], b = c[(r + 1) % 3], d = c[(r + 2) % 3];
		const float target = 0.0f;
		if (code == 1u || code == 2u || code == 4u)
		{
			float l_ab = (target - a.z) / (b.z - a.z);
			float l_ac = (target - a.z) / (d.z - a.z);
			float3 ab = mix3(a, b, l_ab), ac = mix3(a, d, l_ac);
			k0.c[0] = make_float2(ab.x, ab.y); k0.c[1] = make_float2(b.x, b.y); k0.c[2] = make_float2(ac.x, ac.y);
			k1.c[0] = make_float2(ac.x, ac.y); k1.c[1] = make_float2(b.x, b.y); k1.c[2] = make_float2(d.x, d.y);
			dual = true;
		}
		else
		{
			float la = (target - a.z) / (d.z - a.z);
			float lb = (target - b.z) / (d.z - b.z);
			float3 a2 = mix3(a, d, la), b2 = mix3(b, d, lb);
			k0.c[0] = make_float2(a2.x, a2.y); k0.c[1] = make_float2(b2.x, b2.y); k0.c[2] = make_float2(d.x, d.y);
		}
	}
	emit_triangle(count, k0, cull, data);
	if (dual)
		emit_triangle(count, k1, cull, data);
}

// clip a clip-space triangle against w < 1/1024, project, then clip z
__device__ void clip_w_and_emit(uint32_t &count, float4 c0, float4 c1, float4 c2, float cull, float4 *data)
{
	const float MIN_W = 1.0f / 1024.0f;
	float4 c[3] = { c0, c1, c2 };
	uint32_t code = (uint32_t)(c0.w < MIN_W) + (uint32_t)(c1.w < MIN_W) * 2u + (uint32_t)(c2.w < MIN_W) * 4u;
	if (code == 7u)
		return;
	Tri3 k0, k1;
	bool dual = false;
	if (code == 0u)
	{
		k0.c[0] = xyz_div(c0, c0.w);
		k0.c[1] = xyz_div(c1, c1.w);
		k0.c[2] = xyz_div(c2, c2.w);
	}
	else
	{
		int r = (code == 1u || code == 3u) ? 0 : ((code == 2u || code == 6u) ? 1 : 2);
		float4 a = c[r], b = c[(r + 1) % 3], d = c[(r + 2) % 3];
		if (code == 1u || code == 2u || code == 4u)
		{
			float l_ab = (MIN_W - a.w) / (b.w - a.w);
			float l_ac = (MIN_W - a.w) / (d.w - a.w);
			float4 ab = mix4(a, b, l_ab), ac = mix4(a, d, l_ac);
			k0.c[0] = xyz_div(ab, MIN_W); k0.c[1] = xyz_div(b, b.w); k0.c[2] = xyz_div(ac, MIN_W);
			k1.c[0] = xyz_div(ac, MIN_W); k1.c[1] = xyz_div(b, b.w); k1.c[2] = xyz_div(d, d.w);
			dual = true;
		}
		else
		{
			float la = (MIN_W - a.w) / (d.w - a.w);
			float lb = (MIN_W - b.w) / (d.w - b.w);
			float4 a2 = mix4(a, d, la), b2 = mix4(b, d, lb);
			k0.c[0] = xyz_div(a2, MIN_W); k0.c[1] = xyz_div(b2, MIN_W); k0.c[2] = xyz_div(d, d.w);
		}
	}
	clip_z_and_emit(count, k0, cull, data);
	if (dual)
		clip_z_and_emit(count, k1, cull, data);
}

__global__ void __launch_bounds__(64) cull_setup_kernel(CamDev cam, float4 clip_scale, const GrbPositionalLight *__restrict__ lights,
                                                       const uint32_t *__restrict__ type_mask, const float4 *__restrict__ spots, int num_lights,
                                                       float4 *__restrict__ cull_setup)
{
	int index = blockIdx.x * blockDim.x + threadIdx.x;
	if (index >= num_lights)
		return;
	float4 *data = cull_setup + (size_t)index * 32;
	bool point = (__ldg(&type_mask[index >> 5]) >> (index & 31)) & 1u;
	if (point)
	{
		const GrbPositionalLight &l = lights[index];
		float radius = 1.0f / l.inv_radius;
		float4 vw = mul_m4(cam.view, l.position[0], l.position[1], l.position[2], 1.0f);
		float3 view = make_float3(vw.x, -vw.y, -vw.z);
		float2 rx = project_sphere_flat(view.x, view.z, radius);
		float2 ry = project_sphere_flat(view.y, view.z, radius);
		float xy_length = len2(view.x, view.y);
		float ct0, ct1, ct2, ct3;
		if (xy_length < 0.00001f)
		{
			ct0 = 1.0f; ct1 = 0.0f; ct2 = 0.0f; ct3 = 1.0f;
		}
		else
		{
			float inv = 1.0f / xy_length;
			ct0 = view.x * inv; ct1 = -view.y * inv; ct2 = view.y * inv; ct3 = view.x * inv;
		}
		float txy_x = ct0 * view.x + ct2 * view.y;
		float txy_y = ct1 * view.x + ct3 * view.y;
		float2 tx = project_sphere_flat(txy_x, view.z, radius);
		float2 ty = project_sphere_flat(txy_y, view.z, radius);
		bool ellipsis = !isinf(tx.x) && !isinf(tx.y) && !isinf(ty.x) && !isinf(ty.y);
		float cx = (tx.x + tx.y) * 0.5f, cy = (ty.x + ty.y) * 0.5f;
		float erx = tx.y - cx, ery = ty.y - cy;
		data[0] = make_float4(rx.x * clip_scale.x, ry.x * clip_scale.y, rx.y * clip_scale.x, ry.y * clip_scale.y); // ranges.xzyw
		data[1] = make_float4(tx.x, tx.y, ty.x, ty.y);
		data[2] = make_float4(ct0, ct1, ct2, ct3);
		data[3] = make_float4(ellipsis ? 1.0f : 0.0f, 1.0f / erx, 1.0f / ery, 0.0f);
	}
	else
	{
		const float4 *s = spots + (size_t)index * 6;
		float cull = s[5].x;
		uint32_t count = 0xffffffffu;
		if (cull != 0.0f)
		{
			count = 0u;
			float4 c0 = s[0], c1 = s[1], c2 = s[2], c3 = s[3], c4 = s[4];
			clip_w_and_emit(count, c0, c1, c2, cull, data);
			clip_w_and_emit(count, c0, c2, c3, cull, data);
			clip_w_and_emit(count, c0, c3, c4, cull, data);
			clip_w_and_emit(count, c0, c4, c1, cull, data);
			clip_w_and_emit(count, c2, c1, c3, cull, data);
			clip_w_and_emit(count, c4, c3, c1, cull, data);
		}
		reinterpret_cast<uint32_t *>(data)[3] = count; // data[0].w
	}
}

// ------------------------------------------------------------------------------- K3
struct BinParams
{
	float2 inv_res;
	float2 clip_scale_zw;
	int res_x, res_y;
	int num_lights, num_lights_32;
	int first_block_y; // first row of 8x4-tile blocks this launch covers
};

__device__ __forceinline__ bool test_point_light(const BinParams &p, float2 uv, float2 stride, const float4 *__restrict__ d)
{
	float4 e = __ldg(d + 3);
	if (e.x != 0.0f)
	{
		float4 tr = __ldg(d + 1);
		float4 ct = __ldg(d + 2);
		float icx = 0.5f * (tr.x + tr.y), icy = 0.5f * (tr.z + tr.w);
		float lox = uv.x * p.clip_scale_zw.x, loy = uv.y * p.clip_scale_zw.y;
		float hix = (uv.x + stride.x) * p.clip_scale_zw.x, hiy = (uv.y + stride.y) * p.clip_scale_zw.y;
		float d00x = ((ct.x * lox + ct.z * loy) - icx) * e.y, d00y = ((ct.y * lox + ct.w * loy) - icy) * e.z;
		float d01x = ((ct.x * lox + ct.z * hiy) - icx) * e.y, d01y = ((ct.y * lox + ct.w * hiy) - icy) * e.z;
		float d10x = ((ct.x * hix + ct.z * loy) - icx) * e.y, d10y = ((ct.y * hix + ct.w * loy) - icy) * e.z;
		float d11x = ((ct.x * hix + ct.z * hiy) - icx) * e.y, d11y = ((ct.y * hix + ct.w * hiy) - icy) * e.z;
		float max_diag = fmax_(len2(d00x - d11x, d00y - d11y), len2(d01x - d10x, d01y - d10y));
		float min_sq = 1.0f + max_diag;
		min_sq *= min_sq;
		return (d00x * d00x + d00y * d00y) < min_sq && (d01x * d01x + d01y * d01y) < min_sq && (d10x * d10x + d10y * d10y) < min_sq &&
		       (d11x * d11x + d11y * d11y) < min_sq;
	}
	float4 bb = __ldg(d);
	return (uv.x + stride.x > bb.x) && (uv.y + stride.y > bb.y) && (uv.x < bb.z) && (uv.y < bb.w);
}

__device__ __forceinline__ bool test_spot_light(float2 uv, float2 stride, const float4 *__restrict__ d)
{
	uint32_t n = __float_as_uint(__ldg(d).w);
	if (n > kMaxTriangles)
		return true;
	for (uint32_t i = 0; i < n; i++)
	{
		float4 bb = __ldg(d + 4u * i + 3u);
		if ((uv.x + stride.x > bb.x) && (uv.y + stride.y > bb.y) && (uv.x < bb.z) && (uv.y < bb.w))
		{
			float4 base = __ldg(d + 4u * i), dx = __ldg(d + 4u * i + 1u), dy = __ldg(d + 4u * i + 2u);
			float bx = base.x, by = base.y, bz = base.z;
			bx += dx.x * uv.x; by += dx.y * uv.x; bz += dx.z * uv.x;
			bx += dy.x * uv.y; by += dy.y * uv.y; bz += dy.z * uv.y;
			bx += dx.x > 0.0f ? stride.x * dx.x : 0.0f; by += dx.y > 0.0f ? stride.x * dx.y : 0.0f; bz += dx.z > 0.0f ? stride.x * dx.z : 0.0f;
			bx += dy.x > 0.0f ? stride.y * dy.x : 0.0f; by += dy.y > 0.0f ? stride.y * dy.y : 0.0f; bz += dy.z > 0.0f ? stride.y * dy.z : 0.0f;
			if (bx > 0.0f && by > 0.0f && bz > 0.0f)
				return true;
		}
	}
	return false;
}

// One warp per (32-light chunk, 8x4 tile block): lanes first act as the chunk's 32 lights for
// a coarse conservative test of the whole block (ballot), then as the block's 32 tiles for the
// fine test of the surviving lights.  Four warps of a CTA take four consecutive chunks of the
// same tile block so a tile's words leave the CTA as one 16-byte segment.
constexpr int kBinWarps = 4;

// Counted: the list was prepared on the device and holds `*count` lights in its num_lights slots; the chunks at or
// past ceil(count / 32) are stored as zero and the bits >= count are never set.
template <bool Counted>
__global__ void __launch_bounds__(32 * kBinWarps) binning_kernel(BinParams p, const uint32_t *__restrict__ type_mask,
                                                                const float4 *__restrict__ cull_setup, uint32_t *__restrict__ bitmask,
                                                                const int32_t *__restrict__ count)
{
	const int lane = threadIdx.x & 31;
	const int warp = threadIdx.x >> 5;
	const int chunk = blockIdx.x * kBinWarps + warp;
	const int bx = blockIdx.y, by = p.first_block_y + blockIdx.z;
	if (chunk >= p.num_lights_32)
		return;
	if (Counted)
	{
		p.num_lights = min(__ldg(count), p.num_lights);
		if (chunk * 32 >= p.num_lights)
		{
			bitmask[((size_t)(by * 4 + (lane >> 3)) * p.res_x + bx * 8 + (lane & 7)) * p.num_lights_32 + chunk] = 0u;
			return;
		}
	}

	float2 tile_uv = make_float2(2.0f * (float)(bx * 8) * p.inv_res.x - 1.0f, 2.0f * (float)(by * 4) * p.inv_res.y - 1.0f);
	float2 tile_stride = make_float2((2.0f * 8.0f) * p.inv_res.x, (2.0f * 4.0f) * p.inv_res.y);
	const uint32_t tm = __ldg(&type_mask[chunk]);

	bool passed = false;
	{
		int light = chunk * 32 + lane;
		if (light < p.num_lights) // bits >= num_lights are defined 0
		{
			const float4 *d = cull_setup + (size_t)light * 32;
			passed = ((tm >> lane) & 1u) ? test_point_light(p, tile_uv, tile_stride, d) : test_spot_light(tile_uv, tile_stride, d);
		}
	}
	uint32_t ballot = __ballot_sync(0xffffffffu, passed);

	const int px = bx * 8 + (lane & 7), py = by * 4 + (lane >> 3);
	float2 uv = make_float2(2.0f * (float)px * p.inv_res.x - 1.0f, 2.0f * (float)py * p.inv_res.y - 1.0f);
	float2 stride = make_float2(2.0f * p.inv_res.x, 2.0f * p.inv_res.y);
	uint32_t mask = 0u;
	while (ballot)
	{
		int lsb = __ffs(ballot) - 1;
		ballot &= ballot - 1u;
		const float4 *d = cull_setup + (size_t)(chunk * 32 + lsb) * 32;
		bool ok = ((tm >> lsb) & 1u) ? test_point_light(p, uv, stride, d) : test_spot_light(uv, stride, d);
		if (ok)
			mask |= 1u << lsb;
	}
	bitmask[((size_t)py * p.res_x + px) * p.num_lights_32 + chunk] = mask;
}

// ------------------------------------------------------------------------------- K4
// cluster_range[z] = (first, last) light index whose [zmin, zmax] slice range covers z.
// K4 (clusterer_bindless_z_range.comp:20-51): per Z slice, the first and the last light whose slice
// range contains it.  Integer min / max are order-free, so any decomposition gives the reference's
// bits.  One CTA owns 32 consecutive slices -- lane = slice -- and its 32 warps split the light list:
// a warp reads one light's range with a uniform load, skips it when it misses the segment, and
// otherwise every lane updates its own running (first, last) in registers; the warps' partial results
// meet in 64 shared-memory words.  No atomics in the loop, no dynamic shared memory, res_z / 32 CTAs
// instead of one (round 1's single-CTA scatter sat at 0.02 IPC for 25 us).
constexpr int kZSegWarps = 32;

constexpr int kZSegStage = 2048; // light ranges staged per round (16 KiB)

__global__ void __launch_bounds__(32 * kZSegWarps) z_range_segment_kernel(const uint2 *__restrict__ z_ranges, int num_ranges, int res_z,
                                                                         uint2 *__restrict__ cluster_range)
{
	__shared__ uint32_t s_lo[32], s_hi[32];
	__shared__ uint2 s_ranges[kZSegStage];
	__shared__ int s_any;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	if (warp == 0)
	{
		s_lo[lane] = 0xffffffffu;
		s_hi[lane] = 0u;
	}
	const uint32_t seg_lo = blockIdx.x * 32u, seg_hi = seg_lo + 31u;
	const uint32_t z = seg_lo + (uint32_t)lane;
	uint32_t lo = 0xffffffffu, hi = 0u;
	for (int base = 0; base < num_ranges; base += kZSegStage)
	{
		// stage a round of ranges with coalesced loads (a uniform global load per light made the loop a
		// chain of L2 round trips); note whether any of them touches this segment at all
		const int count = min(kZSegStage, num_ranges - base);
		if (threadIdx.x == 0)
			s_any = 0;
		__syncthreads();
		bool touches = false;
		for (int i = threadIdx.x; i < count; i += 32 * kZSegWarps)
		{
			const uint2 r = __ldg(&z_ranges[base + i]);
			s_ranges[i] = r;
			touches |= r.x <= seg_hi && r.y >= seg_lo && r.x <= r.y;
		}
		if (__any_sync(0xffffffffu, touches) && lane == 0)
			s_any = 1;
		__syncthreads();
		if (s_any)
			for (int i = warp; i < count; i += kZSegWarps)
			{
				const uint2 r = s_ranges[i]; // broadcast
				if (z >= r.x && z <= r.y)
				{
					lo = min(lo, (uint32_t)(base + i));
					hi = max(hi, (uint32_t)(base + i));
				}
			}
		__syncthreads();
	}
	if (lo != 0xffffffffu)
	{
		atomicMin(&s_lo[lane], lo);
		atomicMax(&s_hi[lane], hi);
	}
	__syncthreads();
	if (warp == 0 && z < (uint32_t)res_z)
		cluster_range[z] = make_uint2(s_lo[lane], s_hi[lane]);
}

// The reference's per-slice scan (O(res_z * N)); kept as a cross-check (GRB_ZRANGE_SCAN).
__global__ void __launch_bounds__(128) z_range_scan_kernel(const uint2 *__restrict__ z_ranges, int num_ranges, int res_z, uint2 *__restrict__ cluster_range)
{
	uint32_t z = blockIdx.x * blockDim.x + threadIdx.x;
	if (z >= (uint32_t)res_z)
		return;
	uint32_t z_lo = 0xffffffffu, z_hi = 0u;
	for (int i = 0; i < num_ranges; i++)
	{
		uint2 r = __ldg(&z_ranges[i]);
		if (z >= r.x && z <= r.y)
		{
			z_lo = (uint32_t)i;
			break;
		}
	}
	int z_lo_int = max((int)z_lo, 0);
	for (int i = num_ranges - 1; i >= z_lo_int; i--)
	{
		uint2 r = __ldg(&z_ranges[i]);
		if (z >= r.x && z <= r.y)
		{
			z_hi = (uint32_t)i;
			break;
		}
	}
	cluster_range[z] = make_uint2(z_lo, z_hi);
}

CamDev cam_dev(const GrbCamera *c)
{
	CamDev d;
	for (int i = 0; i < 16; i++)
	{
		d.view[i] = c->view[i];
		d.vp[i] = c->view_projection[i];
	}
	d.pos = make_float3(c->camera_position[0], c->camera_position[1], c->camera_position[2]);
	d.front = make_float3(c->camera_front[0], c->camera_front[1], c->camera_front[2]);
	d.z_near = c->z_near;
	d.z_far = c->z_far;
	return d;
}

bool args_ok(const GrbClusterParameters *params, const GrbClusterBuffers *buf, const char *who)
{
	if (!params || !buf || params->num_lights < 0 || params->num_lights_32 != (params->num_lights + 31) / 32 || params->resolution_xy[0] <= 0 ||
	    params->resolution_xy[1] <= 0 || (params->resolution_xy[0] & 7) || (params->resolution_xy[1] & 3))
	{
		set_last_error(who);
		return false;
	}
	return true;
}
} // namespace
} // namespace grb

using namespace grb;

extern "C" int32_t grb_cluster_spot_transform(const GrbCamera *cam, const GrbClusterParameters *params, const GrbClusterBuffers *buf, void *stream)
{
	if (!cam || !args_ok(params, buf, "grb_cluster_spot_transform: bad parameters"))
		return GRB_ERR_INVALID_ARGUMENT;
	int n = params->num_lights;
	if (n == 0)
		return GRB_OK;
	if (!buf->model || !buf->transformed_spots)
	{
		set_last_error("grb_cluster_spot_transform: null model / transformed_spots");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	spot_transform_kernel<<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(cam_dev(cam), buf->model, n, reinterpret_cast<float4 *>(buf->transformed_spots));
	return check_launch("grb_cluster_spot_transform");
}

extern "C" int32_t grb_cluster_cull_setup(const GrbCamera *cam, const GrbClusterParameters *params, const GrbClusterBuffers *buf, void *stream)
{
	if (!cam || !args_ok(params, buf, "grb_cluster_cull_setup: bad parameters"))
		return GRB_ERR_INVALID_ARGUMENT;
	int n = params->num_lights;
	if (n == 0)
		return GRB_OK;
	if (!buf->lights || !buf->type_mask || !buf->transformed_spots || !buf->cull_setup)
	{
		set_last_error("grb_cluster_cull_setup: null buffer");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	float4 cs = make_float4(params->clip_scale[0], params->clip_scale[1], params->clip_scale[2], params->clip_scale[3]);
	cull_setup_kernel<<<(n + 63) / 64, 64, 0, as_stream(stream)>>>(cam_dev(cam), cs, buf->lights, buf->type_mask,
	                                                                reinterpret_cast<const float4 *>(buf->transformed_spots), n,
	                                                                reinterpret_cast<float4 *>(buf->cull_setup));
	return check_launch("grb_cluster_cull_setup");
}

namespace
{
int32_t binning_rows(const GrbClusterParameters *params, const GrbClusterBuffers *buf, const int32_t *count, int32_t tile_y0, int32_t tile_y1, void *stream)
{
	if (!args_ok(params, buf, "grb_cluster_binning: bad parameters (resolution must be a multiple of 8x4)"))
		return GRB_ERR_INVALID_ARGUMENT;
	if (params->num_lights == 0) // update_bindless_mask_buffer_gpu returns early (clusterer.cpp:1466-1467)
		return GRB_OK;
	if (!buf->type_mask || !buf->cull_setup || !buf->bitmask)
	{
		set_last_error("grb_cluster_binning: null buffer");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	BinParams p;
	p.inv_res = make_float2(params->inv_resolution_xy[0], params->inv_resolution_xy[1]);
	p.clip_scale_zw = make_float2(params->clip_scale[2], params->clip_scale[3]);
	p.res_x = params->resolution_xy[0];
	p.res_y = params->resolution_xy[1];
	p.num_lights = params->num_lights;
	p.num_lights_32 = params->num_lights_32;
	// whole blocks of 4 tile rows; an empty or inverted range means every row
	if (tile_y1 <= tile_y0)
	{
		tile_y0 = 0;
		tile_y1 = p.res_y;
	}
	const int by0 = max(tile_y0, 0) / 4, by1 = (min(tile_y1, p.res_y) + 3) / 4;
	if (by1 <= by0)
		return GRB_OK;
	p.first_block_y = by0;
	dim3 grid((p.num_lights_32 + kBinWarps - 1) / kBinWarps, p.res_x / 8, by1 - by0);
	const float4 *cull = reinterpret_cast<const float4 *>(buf->cull_setup);
	if (count)
		binning_kernel<true><<<grid, 32 * kBinWarps, 0, as_stream(stream)>>>(p, buf->type_mask, cull, buf->bitmask, count);
	else
		binning_kernel<false><<<grid, 32 * kBinWarps, 0, as_stream(stream)>>>(p, buf->type_mask, cull, buf->bitmask, nullptr);
	return check_launch("grb_cluster_binning");
}
} // namespace

extern "C" int32_t grb_cluster_binning_rows(const GrbClusterParameters *params, const GrbClusterBuffers *buf, int32_t tile_y0, int32_t tile_y1, void *stream)
{
	return binning_rows(params, buf, nullptr, tile_y0, tile_y1, stream);
}

extern "C" int32_t grb_cluster_binning_rows_counted(const GrbClusterParameters *params, const GrbClusterBuffers *buf, const int32_t *device_count,
                                                    int32_t tile_y0, int32_t tile_y1, void *stream)
{
	if (!device_count)
	{
		set_last_error("grb_cluster_binning_rows_counted: null device_count");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	return binning_rows(params, buf, device_count, tile_y0, tile_y1, stream);
}

extern "C" int32_t grb_cluster_binning(const GrbClusterParameters *params, const GrbClusterBuffers *buf, void *stream)
{
	return grb_cluster_binning_rows(params, buf, 0, 0, stream);
}

extern "C" int32_t grb_cluster_z_range(const GrbClusterBuffers *buf, int32_t num_ranges, void *stream)
{
	if (!buf || !buf->z_ranges || !buf->cluster_range || num_ranges <= 0 || buf->resolution_z <= 0)
	{
		set_last_error("grb_cluster_z_range: null buffer or empty range list (pass one (~0u,0) entry for zero lights)");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	const int res_z = buf->resolution_z;
	static const bool scan = getenv("GRB_ZRANGE_SCAN") != nullptr; // the reference's per-slice scan, for cross-checks
	if (!scan)
		z_range_segment_kernel<<<(res_z + 31) / 32, 32 * kZSegWarps, 0, as_stream(stream)>>>(reinterpret_cast<const uint2 *>(buf->z_ranges), num_ranges, res_z,
		                                                                                    reinterpret_cast<uint2 *>(buf->cluster_range));
	else
		z_range_scan_kernel<<<(res_z + 127) / 128, 128, 0, as_stream(stream)>>>(reinterpret_cast<const uint2 *>(buf->z_ranges), num_ranges, res_z,
		                                                                         reinterpret_cast<uint2 *>(buf->cluster_range));
	return check_launch("grb_cluster_z_range");
}

extern "C" int32_t grb_cluster_build(const GrbCamera *cam, const GrbClusterParameters *params, const GrbClusterBuffers *buf, void *stream)
{
	int32_t r;
	if ((r = grb_cluster_spot_transform(cam, params, buf, stream)) != GRB_OK)
		return r;
	if ((r = grb_cluster_cull_setup(cam, params, buf, stream)) != GRB_OK)
		return r;
	if ((r = grb_cluster_binning(params, buf, stream)) != GRB_OK)
		return r;
	return grb_cluster_z_range(buf, params->num_lights > 0 ? params->num_lights : 1, stream);
}
