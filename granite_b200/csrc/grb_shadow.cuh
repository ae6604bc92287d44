// grb_shadow.cuh -- comparison sampling of the per-light shadow maps (POSITIONAL_LIGHTS_SHADOW with the PCF sampler):
// what the reference's clustering.frag gets from its texture unit through StockSampler::LinearShadow
// (vulkan/device.cpp:1086-1088,1118-1120,1146-1149: compare GREATER_OR_EQUAL, linear, clamp to edge) in
//   spot.h:67-77 + pcf.h:98-99   textureProjLod(sampler2DShadow(uSpotShadowAtlas[index]), shadow[index] * vec4(pos, 1), 0)
//   point.h:45-71                texture(samplerCubeShadow(uPointShadowAtlas[index]), vec4(light_dir_full, shadow_ref))
// CUDA has no comparison sampler and the maps are plain D16_UNORM arrays in HBM (one per light, caller-owned:
// clusterer.cpp:397-407 creates a 2-D image per spot light and a 6-layer cube per point light), so the filter is
// written out: 2 x 2 texels, each compared with the reference depth, blended with the bilinear weights.  Every
// operation is a single IEEE fp32 op in the oracle's order (oracle/oracle_lighting.c, the 2-D and cube samplers there,
// which restates the Vulkan specification's filtering) -- a comparison flips on one ulp of the reference depth, so
// the shadow term is held to the bit-exact bar, not to the lighting pass's one-code bar.  The functions are also
// compiled for the CPU and compared with the oracle (tests/cpp/emulate_shadow.cpp).
#pragma once

#include <stdint.h>

#define GRB_SHADOW_DEV __device__ __forceinline__

namespace grb
{
struct ShadowBilin
{
	int x0, y0;
	float a, b;
};

// oracle_math.h bilin_setup: (u, v) = (s W - 0.5, t H - 0.5), floor + fraction; NaN / huge coordinates stay defined
__device__ __forceinline__ ShadowBilin shadow_bilin(float s, float t, int res)
{
	ShadowBilin r;
	const float fx = __fsub_rn(__fmul_rn(s, (float)res), 0.5f), fy = __fsub_rn(__fmul_rn(t, (float)res), 0.5f);
	float flx = floorf(fx), fly = floorf(fy);
	r.a = __fsub_rn(fx, flx);
	r.b = __fsub_rn(fy, fly);
	flx = fminf(fmaxf(flx, -2.0f), (float)res + 1.0f); // fmaxf / fminf return the non-NaN operand: NaN -> -2
	fly = fminf(fmaxf(fly, -2.0f), (float)res + 1.0f);
	if (!(fx == fx) || (flx != flx))
		flx = 0.0f;
	if (!(fy == fy) || (fly != fly))
		fly = 0.0f;
	r.x0 = (int)flx;
	r.y0 = (int)fly;
	return r;
}

__device__ __forceinline__ float shadow_mix(float c00, float c10, float c01, float c11, float a, float b)
{
	const float ia = __fsub_rn(1.0f, a), ib = __fsub_rn(1.0f, b);
	const float top = __fadd_rn(__fmul_rn(c00, ia), __fmul_rn(c10, a));
	const float bot = __fadd_rn(__fmul_rn(c01, ia), __fmul_rn(c11, a));
	return __fadd_rn(__fmul_rn(top, ib), __fmul_rn(bot, b));
}

__device__ __forceinline__ float shadow_ref_clamp(float ref)
{
	ref = fminf(fmaxf(ref, 0.0f), 1.0f); // fixed-point depth format: D_ref is clamped to [0, 1]
	return ref == ref ? ref : 0.0f;
}

__device__ __forceinline__ float shadow_compare(const uint16_t *map, size_t texel, float ref)
{
	return ref >= __fdiv_rn((float)__ldg(map + texel), 65535.0f) ? 1.0f : 0.0f;
}

// textureProjLod(sampler2DShadow, clip, 0)
__device__ __forceinline__ float shadow_sample_2d(const uint16_t *map, int res, float cx, float cy, float cz, float cw)
{
	const float s = __fdiv_rn(cx, cw), t = __fdiv_rn(cy, cw);
	const float ref = shadow_ref_clamp(__fdiv_rn(cz, cw));
	const ShadowBilin q = shadow_bilin(s, t, res);
	const int x0 = min(max(q.x0, 0), res - 1), x1 = min(max(q.x0 + 1, 0), res - 1);
	const int y0 = min(max(q.y0, 0), res - 1), y1 = min(max(q.y0 + 1, 0), res - 1);
	const size_t r0 = (size_t)y0 * res, r1 = (size_t)y1 * res;
	return shadow_mix(shadow_compare(map, r0 + x0, ref), shadow_compare(map, r0 + x1, ref), shadow_compare(map, r1 + x0, ref),
	                  shadow_compare(map, r1 + x1, ref), q.a, q.b);
}

// SHADOW_MAP_PCF_KERNEL_WIDE (pcf.h:7-80): 6 x 6 texels from the shader's nine comparison gathers (which sit on texel
// corners: exact footprints), weights exp2(-0.375 d^2) (1 - d^2 / 9) per axis, normalised; sums in the shader's order
GRB_SHADOW_DEV float pcf_wide_weight(float p)
{
	const float p2 = __fmul_rn(p, p);
	return __fmul_rn(exp2f(__fmul_rn(p2, -0.375f)), __fsub_rn(1.0f, __fdiv_rn(p2, 9.0f)));
}

GRB_SHADOW_DEV float shadow_sample_2d_wide(const uint16_t *map, int res, float cx, float cy, float cz, float cw)
{
	const float u = __fdiv_rn(cx, cw), v = __fdiv_rn(cy, cw);
	const float ref = shadow_ref_clamp(__fdiv_rn(cz, cw));
	const float fres = (float)res;
	const float ix = __fsub_rn(__fmul_rn(u, fres), 1.5f), iy = __fsub_rn(__fmul_rn(v, fres), 1.5f);
	const float flx = floorf(ix), fly = floorf(iy);
	const float fx = __fsub_rn(ix, flx), fy = __fsub_rn(iy, fly);
	// origin of the first gather's footprint: floor(flx / res * res - 0.5) = flx - 1.  Not clamped to the map: each texel
	// of the 6 x 6 window clamps to the edge on its own, as the gathers' clamp-to-edge does, so near the low edge the
	// window repeats texel 0 as often as it reaches past it.  Beyond 8 texels outside every texel clamps to the same
	// edge, so the bound only keeps the int conversion defined; NaN coordinates give the origin -1.
	const ShadowBilin q = { (int)(flx == flx ? fminf(fmaxf(flx, -8.0f), fres + 8.0f) : 0.0f) - 1,
		                    (int)(fly == fly ? fminf(fmaxf(fly, -8.0f), fres + 8.0f) : 0.0f) - 1, 0.0f, 0.0f };
	float H[6], V[6];
	const float off[6] = { 2.0f, 1.0f, 0.0f, -1.0f, -2.0f, -3.0f };
#pragma unroll
	for (int i = 0; i < 6; i++)
	{
		H[i] = pcf_wide_weight(__fadd_rn(fx, off[i]));
		V[i] = pcf_wide_weight(__fadd_rn(fy, off[i]));
	}
	float var = 0.0f, total_w = 0.0f;
#pragma unroll
	for (int gy = 0; gy < 3; gy++)
	{
		const int p = 2 * gy;
		const size_t r0 = (size_t)min(max(q.y0 + p, 0), res - 1) * res, r1 = (size_t)min(max(q.y0 + p + 1, 0), res - 1) * res;
#pragma unroll
		for (int gx = 0; gx < 3; gx++)
		{
			const int a = 2 * gx;
			const int x0 = min(max(q.x0 + a, 0), res - 1), x1 = min(max(q.x0 + a + 1, 0), res - 1);
			// gather components x = (a, p + 1), y = (a + 1, p + 1), z = (a + 1, p), w = (a, p)
			const float kx = __fmul_rn(H[a], V[p + 1]), ky = __fmul_rn(H[a + 1], V[p + 1]), kz = __fmul_rn(H[a + 1], V[p]), kw = __fmul_rn(H[a], V[p]);
			const float c_x = shadow_compare(map, r1 + x0, ref), c_y = shadow_compare(map, r1 + x1, ref), c_z = shadow_compare(map, r0 + x1, ref),
			            c_w = shadow_compare(map, r0 + x0, ref);
			var = __fadd_rn(var, __fadd_rn(__fadd_rn(__fmul_rn(c_x, kx), __fmul_rn(c_y, ky)), __fadd_rn(__fmul_rn(c_z, kz), __fmul_rn(c_w, kw))));
			total_w = __fadd_rn(total_w, __fadd_rn(__fadd_rn(kx, kz), __fadd_rn(ky, kw)));
		}
	}
	return __fdiv_rn(var, total_w);
}

// Texel (i, j) of face f with i or j possibly one step outside [0, res): the texel across that edge of the cube
// (Vulkan "Cube Map Edge Handling").  Doubled integer coordinates on a cube of half-size res: a texel centre has
// +-res on the major axis and 2 i + 1 - res (|.| < res) in the face; one step outside is +-(res + 1): that axis
// becomes the major one and the old major axis holds the neighbour's edge texel, +-(res - 1).  false at a corner.
__device__ __forceinline__ bool shadow_cube_texel(int res, int f, int i, int j, size_t &texel)
{
	int a = 2 * i + 1 - res, b = 2 * j + 1 - res;
	const bool out_a = a < -res || a > res, out_b = b < -res || b > res;
	if (out_a && out_b)
		return false;
	if (out_a || out_b)
	{
		int x, y, z; // face -> direction: the inverse of the (s_c, t_c, m_a) table
		switch (f)
		{
		case 0: x = res; y = -b; z = -a; break;
		case 1: x = -res; y = -b; z = a; break;
		case 2: x = a; y = res; z = b; break;
		case 3: x = a; y = -res; z = -b; break;
		case 4: x = a; y = -b; z = res; break;
		default: x = -a; y = -b; z = -res; break;
		}
		const int axis = f >> 1; // old major axis
		int *v[3] = { &x, &y, &z };
		*v[axis] = *v[axis] > 0 ? res - 1 : -(res - 1);
#pragma unroll
		for (int k = 0; k < 3; k++)
			if (*v[k] > res || *v[k] < -res)
				*v[k] = *v[k] > 0 ? res : -res;
		if (x == res || x == -res)
		{
			f = x > 0 ? 0 : 1;
			a = x > 0 ? -z : z;
			b = -y;
		}
		else if (y == res || y == -res)
		{
			f = y > 0 ? 2 : 3;
			a = x;
			b = y > 0 ? z : -z;
		}
		else
		{
			f = z > 0 ? 4 : 5;
			a = z > 0 ? x : -x;
			b = -y;
		}
	}
	texel = ((size_t)f * res + (size_t)((b + res - 1) / 2)) * res + (size_t)((a + res - 1) / 2);
	return true;
}

// texture(samplerCubeShadow, vec4(d, ref)); faces in Vulkan layer order +X -X +Y -Y +Z -Z
__device__ __forceinline__ float shadow_sample_cube(const uint16_t *map, int res, float dx, float dy, float dz, float ref)
{
	ref = shadow_ref_clamp(ref);
	const float ax = fabsf(dx), ay = fabsf(dy), az = fabsf(dz);
	int face;
	float sc, tc, ma;
	if (az >= ax && az >= ay)
	{
		face = dz < 0.0f ? 5 : 4;
		sc = dz < 0.0f ? -dx : dx;
		tc = -dy;
		ma = az;
	}
	else if (ay >= ax)
	{
		face = dy < 0.0f ? 3 : 2;
		sc = dx;
		tc = dy < 0.0f ? -dz : dz;
		ma = ay;
	}
	else
	{
		face = dx < 0.0f ? 1 : 0;
		sc = dx < 0.0f ? dz : -dz;
		tc = -dy;
		ma = ax;
	}
	const float s = __fadd_rn(__fmul_rn(0.5f, __fdiv_rn(sc, ma)), 0.5f), t = __fadd_rn(__fmul_rn(0.5f, __fdiv_rn(tc, ma)), 0.5f);
	const ShadowBilin q = shadow_bilin(s, t, res);
	const int x0 = min(max(q.x0, -1), res), x1 = min(max(q.x0 + 1, -1), res);
	const int y0 = min(max(q.y0, -1), res), y1 = min(max(q.y0 + 1, -1), res);
	float c[4];
	bool have[4];
	float sum = 0.0f;
	int n = 0;
#pragma unroll
	for (int k = 0; k < 4; k++)
	{
		size_t texel = 0;
		have[k] = shadow_cube_texel(res, face, (k & 1) ? x1 : x0, (k >> 1) ? y1 : y0, texel);
		c[k] = have[k] ? shadow_compare(map, texel, ref) : 0.0f;
		if (have[k])
		{
			sum = __fadd_rn(sum, c[k]);
			n++;
		}
	}
	if (n == 3)
	{
		const float avg = __fdiv_rn(sum, 3.0f); // the missing corner texel: average of the other three
#pragma unroll
		for (int k = 0; k < 4; k++)
			if (!have[k])
				c[k] = avg;
	}
	return shadow_mix(c[0], c[1], c[2], c[3], q.a, q.b);
}

// spot.h:67-77: clip = shadow[index] * vec4(world_pos, 1) -- (c0 x + c1 y) + (c2 z + c3), the association of the
// reference code as spirv-cross / GLM evaluates it -- then the projective comparison sample
__device__ __forceinline__ float spot_shadow_falloff(const float *m, float px, float py, float pz, const uint16_t *map, int res, bool pcf_wide = false)
{
	float c[4];
#pragma unroll
	for (int r = 0; r < 4; r++)
		c[r] = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + r), px), __fmul_rn(__ldg(m + 4 + r), py)),
		                 __fadd_rn(__fmul_rn(__ldg(m + 8 + r), pz), __ldg(m + 12 + r)));
	return pcf_wide ? shadow_sample_2d_wide(map, res, c[0], c[1], c[2], c[3]) : shadow_sample_2d(map, res, c[0], c[1], c[2], c[3]);
}

// point.h:46-49,67-71: full = world_pos - light_pos; the cube face's depth along its major axis from
// shadow[index][0] = (proj[2].zw, proj[3].zw) (clusterer.cpp:518-521)
__device__ __forceinline__ float point_shadow_falloff(const float *m, float fx, float fy, float fz, const uint16_t *map, int res)
{
	const float max_z = fmaxf(fmaxf(fabsf(fx), fabsf(fy)), fabsf(fz));
	const float rx = __fsub_rn(__ldg(m + 2), __fmul_rn(__ldg(m + 0), max_z)), ry = __fsub_rn(__ldg(m + 3), __fmul_rn(__ldg(m + 1), max_z));
	return shadow_sample_cube(map, res, fx, fy, fz, __fdiv_rn(rx, ry));
}
} // namespace grb
