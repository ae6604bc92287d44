// grb_lighting.cu -- clustered deferred lighting as one sm_90a kernel.
//
// Replaces DeferredLightRenderer::render_light (renderer/renderer.cpp:1004-1156), i.e. the two
// full-screen draws directional.frag and clustering.frag that are additively blended into
// "HDR-main".  Here both happen in ONE pass over the G-buffer: each thread owns one pixel,
// reads its 18 bytes of G-buffer + 4 bytes of HDR once, evaluates the directional light, then
// walks the pixel's light cluster, and writes 4 bytes.  The two blends' intermediate
// B10G11R11 quantisation is reproduced in registers, so the HBM traffic is the compulsory
// 22 B/pixel.
//
// Work mapping: a warp is an 8x4 pixel quad-block (the footprint the reference's fragment
// subgroups have), a CTA is 4 warps side by side (32x4 pixels, so every G-buffer row segment a
// CTA touches is a full 128-byte line).  The light loop is warp-uniform like the reference's
// subgroup-scalarised loop (clusterer_bindless.h:49-81): the warp walks the union of its lanes'
// cluster masks, every lane evaluates the same light (its record is a broadcast load), and a
// lane only ACCUMULATES a light that is in its own (tile, z-slice) mask -- which makes the
// result exactly the per-pixel function, in ascending light order.
//
// Numerics: the cluster indices (tile, z slice) are part of the bit-exact contract, so the
// position reconstruction up to those indices uses non-contracted IEEE ops (fmul/fadd/...).
// The BRDF itself is plain fp32 with FMA and fast reciprocal-sqrt: the result is stored as
// B10G11R11 (6/5 mantissa bits), five orders of magnitude coarser than those rounding
// differences.
#include "grb_common.cuh"
#include "grb_shadow.cuh"

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <mutex>

namespace grb
{
__device__ float g_srgb8_to_linear[256];

namespace
{
constexpr float kPi = 3.1415628f; // assets/shaders/lights/pbr.h:5 (sic)
constexpr float kInvPi = 1.0f / kPi;

struct LightingParams
{
	View<const uint32_t> albedo, normal;
	View<const uint16_t> pbr;
	View<const float> depth;
	View<uint32_t> hdr;
	View<const uint32_t> emissive; // blend destination's initial contents (may be the hdr image itself)
	float ivp[16];
	float3 camera_pos;
	float3 dir_color, dir_dir;
	// cluster
	float3 cbase, cfront;
	float2 xy_scale;
	int res_x, res_y;
	int n32, z_max_index;
	float z_scale;
	float inv_res_x, inv_res_y;
	const GrbPositionalLight *lights;
	const uint32_t *type_mask;
	const uint32_t *bitmask;
	const uint2 *cluster_range;
	int y0, y1;
	// shadowed positional lights (grb_deferred_lighting_shadowed only; grb_shadow.cuh)
	const float *shadow_transforms;    // 16 floats per light: ClustererBindlessTransforms::shadow[index]
	const uint16_t *const *shadow_maps; // per light: D16_UNORM, res^2 (spot) or 6 res^2 (point cube); null = no shadow
	int shadow_res;
	int shadow_pcf_wide; // SHADOW_MAP_PCF_KERNEL_WIDE: spot lights use the 6 x 6 kernel
	// "renderTargetFp16" (scene_viewer_application.cpp:880-884): HDR-main / emissive as R16G16B16A16_SFLOAT; the generic
	// kernel's HDR16 form reads and writes these instead of hdr / emissive
	View<uint2> hdr16;
	View<const uint2> emissive16;
};

struct Surface
{
	float3 pos, N, V;
	float3 F0, one_minus_F0;
	float3 diffuse_k;       // base_color * (1 - metallic) / PI
	float m2_minus_1;       // roughness'^4 - 1
	float c_gd;             // 0.25 * roughness'^4 / PI  (numerator of G*D)
	float one_minus_k, k, Vk; // Schlick-GGX visibility pieces
	float NoV_raw;          // dot(N, V) before the clamp (half-vector algebra)
};

__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

__device__ __forceinline__ uint32_t cluster_mask_range(uint32_t mask, uint32_t rx, uint32_t ry, uint32_t start)
{
	uint32_t hi = start + 32u;
	rx = min(max(rx, start), hi);
	uint32_t ry1 = min(max(ry + 1u, rx), hi);
	uint32_t num_bits = ry1 - rx;
	uint32_t range_mask = num_bits == 32u ? 0xffffffffu : (((1u << num_bits) - 1u) << (rx - start));
	return mask & range_mask;
}

// Cook-Torrance terms shared by the directional and the positional lights (lighting.h:26-46,
// point.h:121-141, spot.h:124-144), arranged for the fewest issue slots -- the pass is bound by
// instruction issue, not by HBM:
//   specular + diffuse = F*G*D + (1-F)*dk = dk + F*(G*D - dk)
//   D*G = (m2 / (PI d^2)) * (0.25 / max(Vk*Lk, 1e-3)),  d = NoH^2 (m2 - 1) + 1
// Returns that sum per channel and NoL; the caller scales by NoL * colour * attenuation.
__device__ __forceinline__ float3 brdf(const Surface &s, float3 L, float &NoL)
{
	// The half vector is formed explicitly: h = V + L.  (|V+L|^2 = 2 + 2 VoL is cheaper by two
	// instructions but loses all precision when L approaches -V: the relative error of the sum is
	// eps/|h|^2, and a bright light at a grazing angle then moves the pixel by several B10G11R11
	// codes.)  With unit V and L: HoV = (1 + VoL)/|h| = |h|/2 and NoL = N.h - N.V.
	float3 h = make_float3(s.V.x + L.x, s.V.y + L.y, s.V.z + L.z);
	float hh = dot3(h, h);
	float inv_h = rsqrt_fast(hh);
	float Nh = dot3(s.N, h);
	NoL = fminf(fmaxf(Nh - s.NoV_raw, 0.001f), 1.0f);
	float NoH = fminf(fmaxf(Nh * inv_h, 0.0001f), 1.0f);
	float f = fminf(fmaf(hh * inv_h, -0.5f, 1.0f), 0.999f); // 1 - max(HoV, 0.001)
	float f2 = f * f;
	float f5 = f2 * f2 * f;
	float d = fmaf(NoH * NoH, s.m2_minus_1, 1.0f);
	// max(Vk * Lk, 1e-3) of the shader is the identity: k = (r' + 1)^2 / 8 >= 0.195 bounds both factors
	float vl = s.Vk * fmaf(NoL, s.one_minus_k, s.k);
	float GD = s.c_gd * rcp_fast(d * d * vl);
	float Fx = fmaf(s.one_minus_F0.x, f5, s.F0.x), Fy = fmaf(s.one_minus_F0.y, f5, s.F0.y), Fz = fmaf(s.one_minus_F0.z, f5, s.F0.z);
	return make_float3(fmaf(Fx, GD - s.diffuse_k.x, s.diffuse_k.x), fmaf(Fy, GD - s.diffuse_k.y, s.diffuse_k.y),
	                   fmaf(Fz, GD - s.diffuse_k.z, s.diffuse_k.z));
}

// Cluster tile column / row of a pixel column / row: the same non-contracted expression the per-pixel
// path below uses (clustering.frag:38, clusterer_bindless.h:39-41), monotone in x and in y.
__device__ __forceinline__ int cluster_tile_x(const LightingParams &p, int x)
{
	return iclamp(__float2int_rz(fmul(fmul(fadd((float)x, 0.5f), p.inv_res_x), p.xy_scale.x)), 0, p.res_x - 1);
}
__device__ __forceinline__ int cluster_tile_y(const LightingParams &p, int y)
{
	return iclamp(__float2int_rz(fmul(fmul(fadd((float)y, 0.5f), p.inv_res_y), p.xy_scale.y)), 0, p.res_y - 1);
}
// order-preserving float <-> unsigned key (for the integer warp reductions)
__device__ __forceinline__ unsigned fkey(float f)
{
	unsigned u = __float_as_uint(f);
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k); }

// Float warp min / max of non-NaN values: sm_90 reduces only integers in one instruction
// (redux.sync.u32), so the floats go through their order-preserving keys.
__device__ __forceinline__ float warp_min_f32(float v) { return fkey_inv(__reduce_min_sync(0xffffffffu, fkey(v))); }
__device__ __forceinline__ float warp_max_f32(float v) { return fkey_inv(__reduce_max_sync(0xffffffffu, fkey(v))); }

// World position of a pixel and its cluster coordinates.  The tile index and Z slice are part
// of the bit-exact contract with the reference (clustering.vert:10-14, clustering.frag:38-39,
// clusterer_bindless.h:39-47), so every op here is a non-contracted IEEE op in a fixed order.
__device__ __forceinline__ float3 reconstruct_position_and_cluster(const LightingParams &p, int x, int y, float depth, int &tile_index, int &z_index)
{
	// vClip = invVP * (ndc.xy, 0, 1) interpolated at the pixel centre, + depth * invVP[2]
	const float ndc_x = fsub(fmul(fmul(2.0f, fadd((float)x, 0.5f)), p.inv_res_x), 1.0f);
	const float ndc_y = fsub(fmul(fmul(2.0f, fadd((float)y, 0.5f)), p.inv_res_y), 1.0f);
	const float *m = p.ivp;
	float cx = fadd(fadd(fadd(fmul(m[0], ndc_x), fmul(m[4], ndc_y)), m[12]), fmul(depth, m[8]));
	float cy = fadd(fadd(fadd(fmul(m[1], ndc_x), fmul(m[5], ndc_y)), m[13]), fmul(depth, m[9]));
	float cz = fadd(fadd(fadd(fmul(m[2], ndc_x), fmul(m[6], ndc_y)), m[14]), fmul(depth, m[10]));
	float cw = fadd(fadd(fadd(fmul(m[3], ndc_x), fmul(m[7], ndc_y)), m[15]), fmul(depth, m[11]));
	float3 pos = make_float3(fdiv(cx, cw), fdiv(cy, cw), fdiv(cz, cw));
	int tx = __float2int_rz(fmul(fmul(fadd((float)x, 0.5f), p.inv_res_x), p.xy_scale.x));
	int ty = __float2int_rz(fmul(fmul(fadd((float)y, 0.5f), p.inv_res_y), p.xy_scale.y));
	tx = iclamp(tx, 0, p.res_x - 1);
	ty = iclamp(ty, 0, p.res_y - 1);
	tile_index = ty * p.res_x + tx;
	float zv = fadd(fadd(fmul(fsub(pos.x, p.cbase.x), p.cfront.x), fmul(fsub(pos.y, p.cbase.y), p.cfront.y)), fmul(fsub(pos.z, p.cbase.z), p.cfront.z));
	z_index = iclamp(__float2int_rz(fmul(zv, p.z_scale)), 0, p.z_max_index);
	return pos;
}

// Diagnostic twin of the lighting kernel's addressing: writes (tile index, z slice) per pixel.
__global__ void __launch_bounds__(128) cluster_indices_kernel(const LightingParams p, int *__restrict__ out_tile, int *__restrict__ out_z)
{
	int x = blockIdx.x * 32 + (threadIdx.x & 31);
	int y = p.y0 + blockIdx.y * 4 + (threadIdx.x >> 5);
	if (x >= p.depth.w || y >= p.y1)
		return;
	float depth = __ldg(&p.depth.at(x, y));
	int tile = -1, z = -1;
	if (depth != 0.0f)
		reconstruct_position_and_cluster(p, x, y, depth, tile, z);
	out_tile[(size_t)y * p.depth.w + x] = tile;
	out_z[(size_t)y * p.depth.w + x] = z;
}

constexpr int kWarpsPerCta = 4;

// SHADOWS: POSITIONAL_LIGHTS_SHADOW (renderer.cpp:369,1126) -- each light's falloff is multiplied by the comparison
// sample of its own shadow map (point.h:45-74, spot.h:51-77), taken only by the lanes the light reaches.
// HDR16: the blend destination is R16G16B16A16_SFLOAT -- each of the two additive blends rounds to fp16 (RNE), alpha
// passes through (the shaders write RGB only).
template <bool SHADOWS, bool HDR16 = false>
__global__ void __launch_bounds__(32 * kWarpsPerCta) deferred_lighting_kernel(const LightingParams p)
{
	__shared__ float s_srgb[256];
	for (int i = threadIdx.x; i < 256; i += blockDim.x)
		s_srgb[i] = g_srgb8_to_linear[i];
	__syncthreads();

	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int x = (blockIdx.x * kWarpsPerCta + warp) * 8 + (lane & 7);
	const int y = p.y0 + blockIdx.y * 4 + (lane >> 3);
	const bool inside = x < p.depth.w && y < p.y1;

	float depth = 0.0f;
	if (inside)
		depth = __ldg(&p.depth.at(x, y));
	// depth test NOT_EQUAL against the quad's z = 0: sky pixels keep the attachment value
	const bool lit = inside && depth != 0.0f;

	Surface s;
	uint32_t dst = 0u;
	float3 dst16 = make_float3(0.f, 0.f, 0.f); // HDR16: the destination's RGB as the fp16 values it holds
	uint32_t alpha16 = 0u;
	uint32_t rx = 0xffffffffu, ry = 0u;
	int cluster_base = 0;
	float3 base_color = make_float3(0.f, 0.f, 0.f);
	if (lit)
	{
		const uint32_t a8 = __ldg(&p.albedo.at(x, y));
		const uint32_t n10 = __ldg(&p.normal.at(x, y));
		const uint32_t mr = __ldg(&p.pbr.at(x, y));
		if (HDR16)
		{
			const uint2 t = __ldg(&p.emissive16.at(x, y));
			const float4 f = unpack_rgba16f(t);
			dst16 = make_float3(f.x, f.y, f.z);
			alpha16 = t.y & 0xffff0000u;
		}
		else
			dst = __ldg(&p.emissive.at(x, y));

		base_color = make_float3(s_srgb[a8 & 0xffu], s_srgb[(a8 >> 8) & 0xffu], s_srgb[(a8 >> 16) & 0xffu]);
		// UNORM decode: these feed only the BRDF (not the bit-exact indices), a multiply by the
		// reciprocal is within half an ulp of the division
		s.N = make_float3(fmaf((float)(n10 & 0x3ffu), 2.0f / 1023.0f, -1.0f), fmaf((float)((n10 >> 10) & 0x3ffu), 2.0f / 1023.0f, -1.0f),
		                  fmaf((float)((n10 >> 20) & 0x3ffu), 2.0f / 1023.0f, -1.0f));
		const float metallic = (float)(mr & 0xffu) * (1.0f / 255.0f);
		const float roughness_in = (float)(mr >> 8) * (1.0f / 255.0f);

		int tile_index, z_index;
		s.pos = reconstruct_position_and_cluster(p, x, y, depth, tile_index, z_index);
		cluster_base = tile_index * p.n32;
		uint2 zr = __ldg(&p.cluster_range[z_index]);
		rx = zr.x;
		ry = zr.y;

		// per-pixel BRDF invariants
		float3 v = make_float3(p.camera_pos.x - s.pos.x, p.camera_pos.y - s.pos.y, p.camera_pos.z - s.pos.z);
		float inv_v = rsqrt_fast(dot3(v, v));
		s.V = make_float3(v.x * inv_v, v.y * inv_v, v.z * inv_v);
		float rough = roughness_in * 0.75f + 0.25f;
		float mm = rough * rough;
		float m2 = mm * mm;
		s.m2_minus_1 = m2 - 1.0f;
		s.c_gd = m2 * (0.25f * kInvPi);
		float r1 = rough + 1.0f;
		s.k = r1 * r1 * 0.125f;
		s.one_minus_k = 1.0f - s.k;
		s.NoV_raw = dot3(s.N, s.V);
		float NoV = fminf(fmaxf(s.NoV_raw, 0.001f), 1.0f);
		s.Vk = NoV * s.one_minus_k + s.k;
		s.F0 = make_float3(0.04f * (1.0f - metallic) + base_color.x * metallic, 0.04f * (1.0f - metallic) + base_color.y * metallic,
		                   0.04f * (1.0f - metallic) + base_color.z * metallic);
		s.one_minus_F0 = make_float3(1.0f - s.F0.x, 1.0f - s.F0.y, 1.0f - s.F0.z);
		float dk = (1.0f - metallic) * kInvPi;
		s.diffuse_k = make_float3(base_color.x * dk, base_color.y * dk, base_color.z * dk);

		// ---- draw 1: directional.frag (LIGHTING_NO_AMBIENT, no shadows, VOLUMETRIC_DIFFUSE_FALLBACK) ----
		float NoL;
		float3 b = brdf(s, p.dir_dir, NoL);
		if (HDR16)
			dst16 = make_float3(h2f(f2h(dst16.x + p.dir_color.x * NoL * b.x + base_color.x * 0.05f)), h2f(f2h(dst16.y + p.dir_color.y * NoL * b.y + base_color.y * 0.05f)),
			                    h2f(f2h(dst16.z + p.dir_color.z * NoL * b.z + base_color.z * 0.05f)));
		else
		{
			float3 e = unpack_r11g11b10(dst);
			dst = pack_r11g11b10(e.x + p.dir_color.x * NoL * b.x + base_color.x * 0.05f, e.y + p.dir_color.y * NoL * b.y + base_color.y * 0.05f,
			                     e.z + p.dir_color.z * NoL * b.z + base_color.z * 0.05f);
		}
	}

	// ---- draw 2: clustering.frag, warp-uniform walk over the union of the lanes' masks ----
	const uint32_t lo_word = rx >> 5, hi_word = ry >> 5; // inactive lanes: (0x7ffffff, 0) => empty
	int z_start = (int)__reduce_min_sync(0xffffffffu, lo_word);
	int z_end = (int)__reduce_max_sync(0xffffffffu, lit ? hi_word : 0u);
	z_end = min(z_end, p.n32 - 1);
	float3 acc = make_float3(0.f, 0.f, 0.f);
	for (int i = z_start; i <= z_end; i++)
	{
		uint32_t own = 0u;
		if (lit && (uint32_t)i >= lo_word && (uint32_t)i <= hi_word)
			own = cluster_mask_range(__ldg(&p.bitmask[cluster_base + i]), rx, ry, 32u * (uint32_t)i);
		uint32_t wmask = __reduce_or_sync(0xffffffffu, own);
		const uint32_t tm = __ldg(&p.type_mask[i]);
		while (wmask)
		{
			const int bit = __ffs(wmask) - 1;
			wmask &= wmask - 1u;
			const float4 *lp = reinterpret_cast<const float4 *>(p.lights + (i * 32 + bit));
			const float4 l1 = __ldg(lp + 1), l2 = __ldg(lp + 2); // position|offset_radius, direction|inv_radius
			float3 l = make_float3(l1.x - s.pos.x, l1.y - s.pos.y, l1.z - s.pos.z);
			float d2 = dot3(l, l);
			// quick reject: beyond the light's radius the falloff is exactly 0 (point.h:41-43); most lights
			// of a 30x34-pixel cluster tile do not reach this 8x4 block, so the warp usually leaves here
			const bool near = ((own >> bit) & 1u) && (d2 * l2.w * l2.w < 1.0f);
			if (!__any_sync(0xffffffffu, near))
				continue;
			const float4 l0 = __ldg(lp); // color|spot scale_bias
			float inv_d = rsqrt_fast(d2);
			float inv_ld = fminf(inv_d, 10.0f); // 1 / max(0.1, dist)
			float xr = fmaxf(0.1f, d2 * inv_d) * l2.w;
			float t = __saturatef(fmaf(xr, 1.0f / (1.0f - 0.9f), -0.9f / (1.0f - 0.9f)));
			float falloff = fmaf(-t * t, fmaf(-2.0f, t, 3.0f), 1.0f);
			float3 L = make_float3(l.x * inv_d, l.y * inv_d, l.z * inv_d);
			if (!((tm >> bit) & 1u))
			{
				// spot.h:34-84: cone term from the packed fp16 scale/bias
				float2 sb = __half22float2(*reinterpret_cast<const __half2 *>(&l0.w));
				float cone_angle = -(L.x * l2.x + L.y * l2.y + L.z * l2.z);
				float cone = __saturatef(fmaf(cone_angle, sb.x, sb.y));
				falloff *= cone * cone;
			}
			if (SHADOWS)
			{
				const int index = i * 32 + bit;
				const uint16_t *map = reinterpret_cast<const uint16_t *>(__ldg(reinterpret_cast<const unsigned long long *>(p.shadow_maps) + index));
				if (map && near && falloff > 0.0f)
				{
					const float *m = p.shadow_transforms + 16 * (size_t)index;
					falloff *= ((tm >> bit) & 1u) ? point_shadow_falloff(m, -l.x, -l.y, -l.z, map, p.shadow_res)
					                              : spot_shadow_falloff(m, s.pos.x, s.pos.y, s.pos.z, map, p.shadow_res, p.shadow_pcf_wide != 0);
				}
			}
			float NoL;
			float3 b = brdf(s, L, NoL);
			float w = NoL * falloff * inv_ld * inv_ld;
			if (near && falloff > 0.0f)
			{
				acc.x = fmaf(l0.x * w, b.x, acc.x);
				acc.y = fmaf(l0.y * w, b.y, acc.y);
				acc.z = fmaf(l0.z * w, b.z, acc.z);
			}
		}
	}

	if (HDR16)
	{
		if (lit)
		{
			uint2 t;
			t.x = (uint32_t)f2h(dst16.x + acc.x) | ((uint32_t)f2h(dst16.y + acc.y) << 16);
			t.y = (uint32_t)f2h(dst16.z + acc.z) | alpha16;
			p.hdr16.at(x, y) = t;
		}
		else if (inside && p.emissive16.p != p.hdr16.p)
			p.hdr16.at(x, y) = __ldg(&p.emissive16.at(x, y)); // sky keeps the attachment value
		return;
	}
	if (lit)
	{
		float3 e = unpack_r11g11b10(dst);
		p.hdr.at(x, y) = pack_r11g11b10(e.x + acc.x, e.y + acc.y, e.z + acc.z);
	}
	else if (inside && p.emissive.p != p.hdr.p)
		p.hdr.at(x, y) = __ldg(&p.emissive.at(x, y)); // sky keeps the attachment value
}
// ---------------------------------------------------------------------------------------------
// Two pixels per thread in float2 lanes.
//
// The pass is bound by instruction issue, and most of the issued instructions are fp32
// multiply/add.  The kernel below carries two horizontally adjacent pixels per thread: the
// per-light control overhead (mask walk, record loads, votes, light-record decoding) is
// amortised over twice the pixels, and the two pixels' vector math (light vector, distances,
// half vector, the three dot products, Fresnel, the GGX terms) gives the scheduler two
// independent dependency chains.  A warp covers a 16x4 pixel block, a CTA 64x4.  Results are
// the same function as the 1-pixel kernel; lanes differ only in fp32 rounding of reassociated
// terms, far below the B10G11R11 step.
using f2 = float2;
__device__ __forceinline__ f2 mk2(float a) { return make_float2(a, a); }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ f2 rsqrt2(f2 a) { return make_float2(rsqrt_fast(a.x), rsqrt_fast(a.y)); }
__device__ __forceinline__ f2 clamp2(f2 a, float lo, float hi) { return make_float2(fminf(fmaxf(a.x, lo), hi), fminf(fmaxf(a.y, lo), hi)); }
__device__ __forceinline__ f2 dot3_2(f2 ax, f2 ay, f2 az, f2 bx, f2 by, f2 bz) { return fma2(az, bz, fma2(ay, by, mul2(ax, bx))); }

struct Surface2
{
	f2 npx, npy, npz; // -position
	f2 Nx, Ny, Nz, Vx, Vy, Vz;
	f2 F0x, F0y, F0z, oFx, oFy, oFz; // F0, 1 - F0
	f2 dkx, dky, dkz, ndkx, ndky, ndkz; // diffuse_k and its negation
	f2 m2m1, cgd, omk, k, Vk, NoVr;
};

// dk + F * (G*D - dk) per channel for both pixels and the (unnormalised) half vector h = V + L; NoL returned for
// the caller's weight.  h is formed explicitly, as in brdf(): from |V+L|^2 = 2 + 2 V.L the grazing specular peak
// (L near -V) loses all precision.
__device__ __forceinline__ void brdf2(const Surface2 &s, f2 hx, f2 hy, f2 hz, f2 &NoL, f2 &tx, f2 &ty, f2 &tz)
{
	f2 hh = dot3_2(hx, hy, hz, hx, hy, hz);
	f2 inv_h = rsqrt2(hh);
	f2 Nh = dot3_2(s.Nx, s.Ny, s.Nz, hx, hy, hz);
	NoL = clamp2(add2(Nh, make_float2(-s.NoVr.x, -s.NoVr.y)), 0.001f, 1.0f); // N.L = N.h - N.V
	f2 NoH = clamp2(mul2(Nh, inv_h), 0.0001f, 1.0f);
	f2 f = fma2(mul2(hh, inv_h), mk2(-0.5f), mk2(1.0f)); // 1 - max(HoV, 0.001), HoV = |h| / 2
	f = make_float2(fminf(f.x, 0.999f), fminf(f.y, 0.999f));
	f2 fsq = mul2(f, f);
	f2 f5 = mul2(mul2(fsq, fsq), f);
	f2 d = fma2(mul2(NoH, NoH), s.m2m1, mk2(1.0f));
	f2 vl = mul2(s.Vk, fma2(NoL, s.omk, s.k)); // >= 0.038, the shader's max(.., 1e-3) is the identity
	f2 den = mul2(mul2(d, d), vl);
	f2 GD = mul2(s.cgd, make_float2(rcp_fast(den.x), rcp_fast(den.y)));
	f2 Fx = fma2(s.oFx, f5, s.F0x), Fy = fma2(s.oFy, f5, s.F0y), Fz = fma2(s.oFz, f5, s.F0z);
	tx = fma2(Fx, add2(GD, s.ndkx), s.dkx);
	ty = fma2(Fy, add2(GD, s.ndky), s.dky);
	tz = fma2(Fz, add2(GD, s.ndkz), s.dkz);
}

struct PixelSetup
{
	bool lit;
	uint32_t dst, rx, ry;
	int cluster_base;
	float3 pos, N, V, F0, dk, base_color;
	float m2m1, cgd, omk, k, Vk, NoVr;
};

// Everything the 1-pixel kernel does before its light loop, for one pixel.
__device__ __forceinline__ PixelSetup setup_pixel(const LightingParams &p, const float *s_srgb, int x, int y, bool inside, float depth, uint32_t a8,
                                                 uint32_t n10, uint32_t mr, uint32_t emissive)
{
	PixelSetup q;
	q.lit = inside && depth != 0.0f;
	q.dst = emissive;
	q.rx = 0xffffffffu;
	q.ry = 0u;
	q.cluster_base = 0;
	q.pos = q.N = q.V = q.F0 = q.dk = q.base_color = make_float3(0.f, 0.f, 0.f);
	q.m2m1 = q.cgd = q.omk = q.k = q.Vk = q.NoVr = 0.0f;
	if (!q.lit)
		return q;
	q.base_color = make_float3(s_srgb[a8 & 0xffu], s_srgb[(a8 >> 8) & 0xffu], s_srgb[(a8 >> 16) & 0xffu]);
	q.N = make_float3(fmaf((float)(n10 & 0x3ffu), 2.0f / 1023.0f, -1.0f), fmaf((float)((n10 >> 10) & 0x3ffu), 2.0f / 1023.0f, -1.0f),
	                  fmaf((float)((n10 >> 20) & 0x3ffu), 2.0f / 1023.0f, -1.0f));
	const float metallic = (float)(mr & 0xffu) * (1.0f / 255.0f);
	const float roughness_in = (float)(mr >> 8) * (1.0f / 255.0f);
	int tile_index, z_index;
	q.pos = reconstruct_position_and_cluster(p, x, y, depth, tile_index, z_index);
	q.cluster_base = tile_index * p.n32;
	uint2 zr = __ldg(&p.cluster_range[z_index]);
	q.rx = zr.x;
	q.ry = zr.y;
	float3 v = make_float3(p.camera_pos.x - q.pos.x, p.camera_pos.y - q.pos.y, p.camera_pos.z - q.pos.z);
	float inv_v = rsqrt_fast(dot3(v, v));
	q.V = make_float3(v.x * inv_v, v.y * inv_v, v.z * inv_v);
	float rough = roughness_in * 0.75f + 0.25f;
	float mm = rough * rough;
	float m2 = mm * mm;
	q.m2m1 = m2 - 1.0f;
	q.cgd = m2 * (0.25f * kInvPi);
	float r1 = rough + 1.0f;
	q.k = r1 * r1 * 0.125f;
	q.omk = 1.0f - q.k;
	q.NoVr = dot3(q.N, q.V);
	float NoV = fminf(fmaxf(q.NoVr, 0.001f), 1.0f);
	q.Vk = NoV * q.omk + q.k;
	q.F0 = make_float3(0.04f * (1.0f - metallic) + q.base_color.x * metallic, 0.04f * (1.0f - metallic) + q.base_color.y * metallic,
	                   0.04f * (1.0f - metallic) + q.base_color.z * metallic);
	float dk = (1.0f - metallic) * kInvPi;
	q.dk = make_float3(q.base_color.x * dk, q.base_color.y * dk, q.base_color.z * dk);
	return q;
}

// G-buffer fetch + per-pixel invariants for the pixel pair (x, x + 1) of row y.
struct PairSetup
{
	PixelSetup A, B;
	Surface2 s;
	int z_start, z_end; // the warp's range of 32-light words (empty when z_end < z_start)
};

__device__ __forceinline__ void setup_pair(const LightingParams &p, const float *s_srgb, int x, int y, bool inside, PairSetup &q)
{
	float2 depth = make_float2(0.f, 0.f);
	uint2 a8 = make_uint2(0u, 0u), n10 = make_uint2(0u, 0u), em = make_uint2(0u, 0u);
	uint32_t mr2 = 0u;
	if (inside)
	{
		depth = __ldg(reinterpret_cast<const float2 *>(&p.depth.at(x, y)));
		// not gated on depth != 0: a dependent second round trip to HBM costs more than the sky's bytes
		a8 = __ldg(reinterpret_cast<const uint2 *>(&p.albedo.at(x, y)));
		n10 = __ldg(reinterpret_cast<const uint2 *>(&p.normal.at(x, y)));
		mr2 = __ldg(reinterpret_cast<const uint32_t *>(&p.pbr.at(x, y)));
		em = __ldg(reinterpret_cast<const uint2 *>(&p.emissive.at(x, y)));
	}
	q.A = setup_pixel(p, s_srgb, x, y, inside, depth.x, a8.x, n10.x, mr2 & 0xffffu, em.x);
	q.B = setup_pixel(p, s_srgb, x + 1, y, inside, depth.y, a8.y, n10.y, mr2 >> 16, em.y);
	const PixelSetup &A = q.A, &B = q.B;
	Surface2 &s = q.s;
	s.npx = make_float2(-A.pos.x, -B.pos.x); s.npy = make_float2(-A.pos.y, -B.pos.y); s.npz = make_float2(-A.pos.z, -B.pos.z);
	s.Nx = make_float2(A.N.x, B.N.x); s.Ny = make_float2(A.N.y, B.N.y); s.Nz = make_float2(A.N.z, B.N.z);
	s.Vx = make_float2(A.V.x, B.V.x); s.Vy = make_float2(A.V.y, B.V.y); s.Vz = make_float2(A.V.z, B.V.z);
	s.F0x = make_float2(A.F0.x, B.F0.x); s.F0y = make_float2(A.F0.y, B.F0.y); s.F0z = make_float2(A.F0.z, B.F0.z);
	s.oFx = make_float2(1.0f - A.F0.x, 1.0f - B.F0.x); s.oFy = make_float2(1.0f - A.F0.y, 1.0f - B.F0.y); s.oFz = make_float2(1.0f - A.F0.z, 1.0f - B.F0.z);
	s.dkx = make_float2(A.dk.x, B.dk.x); s.dky = make_float2(A.dk.y, B.dk.y); s.dkz = make_float2(A.dk.z, B.dk.z);
	s.ndkx = make_float2(-A.dk.x, -B.dk.x); s.ndky = make_float2(-A.dk.y, -B.dk.y); s.ndkz = make_float2(-A.dk.z, -B.dk.z);
	s.m2m1 = make_float2(A.m2m1, B.m2m1); s.cgd = make_float2(A.cgd, B.cgd);
	s.omk = make_float2(A.omk, B.omk); s.k = make_float2(A.k, B.k); s.Vk = make_float2(A.Vk, B.Vk);
	s.NoVr = make_float2(A.NoVr, B.NoVr);
	const uint32_t loA = A.rx >> 5, hiA = A.ry >> 5, loB = B.rx >> 5, hiB = B.ry >> 5; // unlit: (0x7ffffff, 0) => empty
	q.z_start = (int)__reduce_min_sync(0xffffffffu, min(loA, loB));
	q.z_end = min((int)__reduce_max_sync(0xffffffffu, max(A.lit ? hiA : 0u, B.lit ? hiB : 0u)), p.n32 - 1);
}

// draw 2 (clustering.frag): warp-uniform walk over the union of all 64 pixels' masks, words
// first, first + step, ... <= q.z_end; adds the lights' contribution to (accx, accy, accz).
__device__ __forceinline__ void walk_lights(const LightingParams &p, const PairSetup &q, int first, int step, float4 (*staged)[32], f2 &accx, f2 &accy,
                                            f2 &accz)
{
	const int lane = threadIdx.x & 31;
	const PixelSetup &A = q.A, &B = q.B;
	const Surface2 &s = q.s;
	const uint32_t loA = A.rx >> 5, hiA = A.ry >> 5, loB = B.rx >> 5, hiB = B.ry >> 5;
	for (int i = first; i <= q.z_end; i += step)
	{
		uint32_t ownA = 0u, ownB = 0u;
		if (A.lit && (uint32_t)i >= loA && (uint32_t)i <= hiA)
			ownA = cluster_mask_range(__ldg(&p.bitmask[A.cluster_base + i]), A.rx, A.ry, 32u * (uint32_t)i);
		if (B.lit && (uint32_t)i >= loB && (uint32_t)i <= hiB)
			ownB = cluster_mask_range(__ldg(&p.bitmask[B.cluster_base + i]), B.rx, B.ry, 32u * (uint32_t)i);
		uint32_t wmask = __reduce_or_sync(0xffffffffu, ownA | ownB);
		if (!wmask)
			continue;
		const uint32_t tm = __ldg(&p.type_mask[i]);
		// Stage the word's records in shared memory, lane b fetching light 32 i + b: one parallel trip
		// to L1/L2 per word.  Reading each record with a broadcast load right before its first use
		// (one dependent trip per light) was the largest stall in light-dense regions.
		__syncwarp();
		if ((wmask >> lane) & 1u)
		{
			const float4 *mine = reinterpret_cast<const float4 *>(p.lights + (i * 32 + lane));
			staged[0][lane] = __ldg(mine);
			staged[1][lane] = __ldg(mine + 1);
			staged[2][lane] = __ldg(mine + 2);
		}
		__syncwarp();
		while (wmask)
		{
			const int bit = __ffs(wmask) - 1;
			wmask &= wmask - 1u;
			const float4 l1 = staged[1][bit], l2 = staged[2][bit]; // position|offset_radius, direction|inv_radius
			f2 lx = add2(mk2(l1.x), s.npx), ly = add2(mk2(l1.y), s.npy), lz = add2(mk2(l1.z), s.npz);
			f2 d2 = dot3_2(lx, ly, lz, lx, ly, lz);
			const float inv_r2 = l2.w * l2.w;
			const bool nearA = ((ownA >> bit) & 1u) && (d2.x * inv_r2 < 1.0f);
			const bool nearB = ((ownB >> bit) & 1u) && (d2.y * inv_r2 < 1.0f);
			// quick reject: beyond the light's radius the falloff is exactly 0 (point.h:41-43)
			if (!__any_sync(0xffffffffu, nearA || nearB))
				continue;
			const float4 l0 = staged[0][bit]; // color|spot scale_bias
			f2 inv_d = rsqrt2(d2);
			f2 inv_ld = make_float2(fminf(inv_d.x, 10.0f), fminf(inv_d.y, 10.0f));
			f2 dist = mul2(d2, inv_d);
			f2 xr = mul2(make_float2(fmaxf(dist.x, 0.1f), fmaxf(dist.y, 0.1f)), mk2(l2.w));
			f2 t = fma2(xr, mk2(1.0f / (1.0f - 0.9f)), mk2(-0.9f / (1.0f - 0.9f)));
			t = make_float2(__saturatef(t.x), __saturatef(t.y));
			f2 falloff = fma2(mul2(mul2(t, t), fma2(mk2(-2.0f), t, mk2(3.0f))), mk2(-1.0f), mk2(1.0f));
			if (!((tm >> bit) & 1u))
			{
				float2 sb = __half22float2(*reinterpret_cast<const __half2 *>(&l0.w));
				f2 cone_angle = mul2(dot3_2(lx, ly, lz, mk2(l2.x), mk2(l2.y), mk2(l2.z)), inv_d);
				f2 cone = fma2(cone_angle, mk2(-sb.x), mk2(sb.y));
				cone = make_float2(__saturatef(cone.x), __saturatef(cone.y));
				falloff = mul2(falloff, mul2(cone, cone));
			}
			f2 NoL, tx, ty, tz;
			brdf2(s, fma2(lx, inv_d, s.Vx), fma2(ly, inv_d, s.Vy), fma2(lz, inv_d, s.Vz), NoL, tx, ty, tz);
			f2 w = mul2(mul2(NoL, falloff), mul2(inv_ld, inv_ld));
			// a lane outside the light's mask or radius adds exactly 0 (falloff is 0 beyond the radius)
			w = make_float2(nearA ? w.x : 0.0f, nearB ? w.y : 0.0f);
			accx = fma2(mul2(mk2(l0.x), w), tx, accx);
			accy = fma2(mul2(mk2(l0.y), w), ty, accy);
			accz = fma2(mul2(mk2(l0.z), w), tz, accz);
		}
	}
}

__global__ void __launch_bounds__(32 * kWarpsPerCta, 5) deferred_lighting2_kernel(const LightingParams p)
{
	__shared__ float s_srgb[256];
	for (int i = threadIdx.x; i < 256; i += blockDim.x)
		s_srgb[i] = g_srgb8_to_linear[i];
	__syncthreads();

	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int x = ((blockIdx.x * kWarpsPerCta + warp) * 8 + (lane & 7)) * 2; // pixels x and x + 1 (width is even on this path)
	const int y = p.y0 + blockIdx.y * 4 + (lane >> 3);
	const bool inside = x < p.hdr.w && y < p.y1;

	__shared__ float4 s_lights[kWarpsPerCta][3][32];
	PairSetup q;
	setup_pair(p, s_srgb, x, y, inside, q);
	const PixelSetup &A = q.A, &B = q.B;

	// ---- draw 1: directional light for both pixels ----
	uint32_t dstA = A.dst, dstB = B.dst;
	{
		const Surface2 &s = q.s;
		f2 NoL, tx, ty, tz;
		const f2 dx = mk2(p.dir_dir.x), dy = mk2(p.dir_dir.y), dz = mk2(p.dir_dir.z);
		brdf2(s, add2(s.Vx, dx), add2(s.Vy, dy), add2(s.Vz, dz), NoL, tx, ty, tz);
		if (A.lit)
		{
			float3 e = unpack_r11g11b10(dstA);
			dstA = pack_r11g11b10(e.x + p.dir_color.x * NoL.x * tx.x + A.base_color.x * 0.05f, e.y + p.dir_color.y * NoL.x * ty.x + A.base_color.y * 0.05f,
			                      e.z + p.dir_color.z * NoL.x * tz.x + A.base_color.z * 0.05f);
		}
		if (B.lit)
		{
			float3 e = unpack_r11g11b10(dstB);
			dstB = pack_r11g11b10(e.x + p.dir_color.x * NoL.y * tx.y + B.base_color.x * 0.05f, e.y + p.dir_color.y * NoL.y * ty.y + B.base_color.y * 0.05f,
			                      e.z + p.dir_color.z * NoL.y * tz.y + B.base_color.z * 0.05f);
		}
	}

	// ---- draw 2 ----
	// (Handing the light-dense blocks -- hundreds of lights per pixel, one warp busy for ~100 us --
	// to a second kernel that spreads a block's lights over four warps was tried: bit-compatible,
	// but the frame got 9 % slower, because the dense blocks then no longer overlap the cheap ones.)
	f2 accx = mk2(0.0f), accy = mk2(0.0f), accz = mk2(0.0f);
	walk_lights(p, q, q.z_start, 1, s_lights[warp], accx, accy, accz);
	const float3 accA = make_float3(accx.x, accy.x, accz.x), accB = make_float3(accx.y, accy.y, accz.y);

	if (inside)
	{
		uint2 out = make_uint2(dstA, dstB);
		if (A.lit)
		{
			float3 e = unpack_r11g11b10(dstA);
			out.x = pack_r11g11b10(e.x + accA.x, e.y + accA.y, e.z + accA.z);
		}
		if (B.lit)
		{
			float3 e = unpack_r11g11b10(dstB);
			out.y = pack_r11g11b10(e.x + accB.x, e.y + accB.y, e.z + accB.z);
		}
		// sky pixels carry the emissive value through (identical bits when blending in place)
		if (A.lit || B.lit || p.emissive.p != p.hdr.p)
			*reinterpret_cast<uint2 *>(&p.hdr.at(x, y)) = out;
	}
}

// ---------------------------------------------------------------------------------------------
// Persistent form: one 512-thread CTA per SM, the frame's light table resident in shared memory.
//
// What bounded the kernel above in the light-dense rows (100-230 lights per pixel) was not issue
// slots but a chain of dependent round trips per 32-light word: bitmask word (L2) -> warp OR ->
// records (L2) -> per light: distance, vote, branch.  Here
//   * the whole light table (48 B x 4096 = 192 KiB) is copied ONCE per CTA into shared memory by
//     the bulk-copy engine (cp.async.bulk, one mbarrier) while the first pixel blocks are being
//     set up; every record read after that is a shared-memory broadcast;
//   * a warp first builds the list of lights that can reach its 16x4 pixel block: the bitmask rows
//     of the (<= 4) cluster tiles under the block are read lane-parallel (lane j owns words j,
//     j + 32, ...), cut to the hull of the pixels' Z-slice ranges, and each candidate is tested
//     by its own lane against the block's world-space bounding box (sphere-box distance);
//     ballots compact the survivors, in ascending light order, into a per-warp list;
//   * the list is then shaded two lights per iteration -- two independent dependency chains --
//     with no votes, branches or mask tests inside: a light that does not reach a pixel adds
//     exactly 0 there because the smoothstep range falloff (point.h:41-43) is exactly 0 beyond
//     the radius, which is the invariant the clusterer is built on;
//   * the sums over lights are kept as  S1 = sum c w (1-f5),  S2 = sum c G w (1-f5),
//     S3 = sum c G w f5  (c colour, w = NoL falloff / d^2, f5 the Schlick weight, G = D*Vis), so
//     that F0 and the diffuse colour leave the loop:  result = dk (1-F0) S1 + F0 S2 + S3;
//   * pixel blocks are handed out through an atomic queue in chunks, so a warp that drew cheap
//     blocks simply draws more.
#ifndef GRB_LIGHTING_WARPS
#define GRB_LIGHTING_WARPS 16
#endif
constexpr int kPWarps = GRB_LIGHTING_WARPS;      // 16: two lights per iteration, 128 registers; 20: one light, <= 102 registers
constexpr bool kPairLights = kPWarps <= 16;
constexpr unsigned kSlotBytes = kPWarps > 16 ? 40u : 48u; // G-buffer prefetch slot per thread (36 bytes used)
constexpr int kListCap = kPWarps > 16 ? 128 : 160; // light list entries per warp; shaded in batches when it fills up
constexpr int kMaxOrderRows = kPWarps > 16 ? 1024 : 2048; // block rows whose schedule fits in shared memory (images up to 4096 / 8192 rows)

#ifdef GRB_LIGHTING_DEBUG
constexpr int kDbgBlocks = 240 * 540;
__device__ uint2 g_dbg_block[kDbgBlocks];   // (cycles, start ns since this warp's start)
__device__ uint2 g_dbg_warp_end[256 * 16];  // (warp start ns low bits, ns from warp start to warp end)
__device__ unsigned long long g_dbg_t0;
__device__ unsigned g_dbg_warp_items[256 * 16];
__device__ uint2 g_dbg_warp_last[256 * 16][8]; // ring of the last 8 (item, fetch time ns) per warp
__device__ __forceinline__ unsigned long long globaltimer_ns()
{
	unsigned long long t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return t;
}
#endif

struct QueueSlot
{
	unsigned next_block;
	unsigned ctas_done;
};
__device__ QueueSlot g_light_queue[64];

struct PersistentArgs
{
	QueueSlot *queue;
	int blocks_x, blocks_y, total_items; // total_items = blocks_x * blocks_y
	int n_lights;
	uint32_t *schedule; // optional: [blocks_x, blocks_y, valid, 0][max block cost per strip][strips by falling cost]
	unsigned rec_bytes; // n_lights * 48, multiple of 16
};

struct SurfaceP
{
	f2 npx, npy, npz; // -position
	f2 Nx, Ny, Nz, Vx, Vy, Vz;
	f2 m2m1, cgd, omk, k, Vk, nNoVr; // nNoVr = -dot(N, V)
};

__device__ __forceinline__ f2 rcp2(f2 a) { return make_float2(rcp_fast(a.x), rcp_fast(a.y)); }
__device__ __forceinline__ f2 min2(f2 a, float hi) { return make_float2(fminf(a.x, hi), fminf(a.y, hi)); }
__device__ __forceinline__ f2 max2(f2 a, float lo) { return make_float2(fmaxf(a.x, lo), fmaxf(a.y, lo)); }
__device__ __forceinline__ f2 sat2(f2 a) { return make_float2(__saturatef(a.x), __saturatef(a.y)); }

// Per light and pixel pair: a = w (1 - f5), G a, G f5 w  for the (unnormalised) half vector h = V + L
// and the attenuation w_pre (everything of the weight except NoL).
__device__ __forceinline__ void shade_terms(const SurfaceP &s, f2 hx, f2 hy, f2 hz, f2 w_pre, f2 &a, f2 &ga, f2 &gb)
{
	f2 hh = dot3_2(hx, hy, hz, hx, hy, hz);
	f2 inv_h = rsqrt2(hh);
	f2 Nh = dot3_2(s.Nx, s.Ny, s.Nz, hx, hy, hz);
	f2 NoH = clamp2(mul2(Nh, inv_h), 0.0001f, 1.0f);
	f2 NoL = clamp2(add2(Nh, s.nNoVr), 0.001f, 1.0f);          // N.L = N.h - N.V
	f2 f = min2(fma2(mul2(hh, inv_h), mk2(-0.5f), mk2(1.0f)), 0.999f); // 1 - max(HoV, 0.001), HoV = |h| / 2
	f2 fsq = mul2(f, f);
	f2 f5 = mul2(mul2(fsq, fsq), f);
	f2 d = fma2(mul2(NoH, NoH), s.m2m1, mk2(1.0f));
	f2 vl = mul2(s.Vk, fma2(NoL, s.omk, s.k)); // >= 0.038: the shader's max(.., 1e-3) is the identity
	f2 g = mul2(s.cgd, rcp2(mul2(mul2(d, d), vl)));
	f2 w = mul2(NoL, w_pre);
	f2 b = mul2(w, f5);
	a = fma2(b, mk2(-1.0f), w);
	ga = mul2(g, a);
	gb = mul2(g, b);
}

// point.h:33-81 / spot.h:34-84 for one light record and the pixel pair, then shade_terms.
// SPOTS = false: both lights of the iteration are point lights (straight-line code, the two
// calls interleave freely); SPOTS = true: the cone term is computed and selected per light.
template <bool SPOTS>
__device__ __forceinline__ void light_terms(const SurfaceP &s, const float4 l0, const float4 l1, const float4 l2, bool is_spot, f2 &a, f2 &ga, f2 &gb)
{
	f2 lx = add2(mk2(l1.x), s.npx), ly = add2(mk2(l1.y), s.npy), lz = add2(mk2(l1.z), s.npz);
	f2 d2 = dot3_2(lx, ly, lz, lx, ly, lz);
	f2 inv_d = rsqrt2(d2);
	f2 inv_ld = min2(inv_d, 10.0f); // 1 / max(0.1, dist)
	f2 xr = mul2(max2(mul2(d2, inv_d), 0.1f), mk2(l2.w));
	f2 t = sat2(fma2(xr, mk2(1.0f / (1.0f - 0.9f)), mk2(-0.9f / (1.0f - 0.9f))));
	f2 falloff = fma2(mul2(mul2(t, t), fma2(mk2(-2.0f), t, mk2(3.0f))), mk2(-1.0f), mk2(1.0f));
	if (SPOTS)
	{
		float2 sb = __half22float2(*reinterpret_cast<const __half2 *>(&l0.w));
		f2 cone_angle = mul2(dot3_2(lx, ly, lz, mk2(l2.x), mk2(l2.y), mk2(l2.z)), inv_d);
		f2 cone = sat2(fma2(cone_angle, mk2(-sb.x), mk2(sb.y)));
		cone = mul2(cone, cone);
		falloff = mul2(falloff, is_spot ? cone : mk2(1.0f));
	}
	f2 w_pre = mul2(falloff, mul2(inv_ld, inv_ld));
	shade_terms(s, fma2(lx, inv_d, s.Vx), fma2(ly, inv_d, s.Vy), fma2(lz, inv_d, s.Vz), w_pre, a, ga, gb);
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Where the persistent kernel's 4-row work items (strips) lie.  Strip i of a band: rows from p.y0 + 4 i.
struct BandStrips
{
	__device__ __forceinline__ int first_row(const LightingParams &p, int strip) const { return p.y0 + strip * 4; }
};
// Strip i of a stripe set (grb_deferred_lighting_stripes): stripe k = i / strips_per_stripe starts at first + k period,
// and the strip lies (i mod strips_per_stripe) * 4 rows into it.  Only the last stripe can be cut by the image (p.y1).
struct StripeSetStrips
{
	int first, strips_per_stripe, period;
	__device__ __forceinline__ int first_row(const LightingParams &, int strip) const
	{
		const int k = strip / strips_per_stripe;
		return first + k * period + (strip - k * strips_per_stripe) * 4;
	}
};

// Strips: BandStrips (the rows p.y0 .. p.y1) or StripeSetStrips (grb_deferred_lighting_stripes).
template <class Strips>
__global__ void __launch_bounds__(32 * kPWarps, 1) deferred_lighting_persistent_kernel(const LightingParams p, const PersistentArgs a, const Strips strips)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	// layout: [records (n_lights + 1) x 48 B][srgb LUT 1 KiB][lists kPWarps x (kListCap + 2) u16][G-buffer prefetch slots][mbarrier]
	float4 *s_rec = reinterpret_cast<float4 *>(smem_raw);
	const unsigned rec_total = a.rec_bytes + 48u;
	float *s_srgb = reinterpret_cast<float *>(smem_raw + rec_total);
	uint16_t *s_lists = reinterpret_cast<uint16_t *>(smem_raw + rec_total + 1024u);
	const unsigned lists_bytes = (kPWarps * (kListCap + 2) * 2u + 15u) & ~15u;
	unsigned char *s_prefetch = smem_raw + rec_total + 1024u + lists_bytes; // 48 B per thread
	uint64_t *s_bar = reinterpret_cast<uint64_t *>(s_prefetch + 32u * kPWarps * kSlotBytes);
	uint16_t *s_order = reinterpret_cast<uint16_t *>(s_bar + 2); // kMaxOrderRows entries

	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t bar = smem_u32(s_bar);
	if (threadIdx.x == 0)
	{
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		// the dummy record that pads an odd batch: black, infinitely far away, falloff exactly 0
		s_rec[3 * a.n_lights + 0] = make_float4(0.f, 0.f, 0.f, 0.f);
		s_rec[3 * a.n_lights + 1] = make_float4(1.0e18f, 0.f, 0.f, 0.f);
		s_rec[3 * a.n_lights + 2] = make_float4(0.f, 0.f, 1.f, 1.f);
	}
	for (int i = threadIdx.x; i < 256; i += blockDim.x)
		s_srgb[i] = g_srgb8_to_linear[i];
	// Block rows in the order of falling cost, as measured by the previous launch on the same
	// schedule buffer (longest-processing-time-first: the queue then ends on the cheapest rows and
	// no warp is left holding an expensive block while the others have run dry).
	const bool scheduled = a.schedule && a.blocks_y <= kMaxOrderRows && a.schedule[0] == (uint32_t)a.blocks_x &&
	                       a.schedule[1] == (uint32_t)a.blocks_y && a.schedule[2] == 1u;
	if (scheduled)
		for (int i = threadIdx.x; i < a.blocks_y; i += blockDim.x)
			s_order[i] = (uint16_t)a.schedule[4 + a.blocks_y + i];
	__syncthreads();
	// the light table (16-byte aligned, launch_deferred_lighting checks it) by the bulk-copy engine
	if (threadIdx.x == 0 && a.rec_bytes)
	{
		asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(a.rec_bytes) : "memory");
		const unsigned char *src = reinterpret_cast<const unsigned char *>(p.lights);
		for (unsigned off = 0; off < a.rec_bytes; off += 32768u)
		{
			const unsigned n = min(32768u, a.rec_bytes - off);
			asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_raw + off)),
			             "l"(src + off), "r"(n), "r"(bar)
			             : "memory");
		}
	}
	bool table_ready = a.rec_bytes == 0;

	uint16_t *list = s_lists + warp * (kListCap + 2);
	const unsigned dummy_entry = (unsigned)a.n_lights;
	const unsigned lt_mask = (1u << lane) - 1u;
	const unsigned total = (unsigned)a.total_items;
	const unsigned n_warps = gridDim.x * kPWarps;

	// Work items are 16x4-pixel blocks (lane = 8 x 4 pixel pairs), a.blocks_x = ceil(w / 16) per strip (4 pixel
	// rows), strip by strip in schedule order, one item per atomic.
	//
	// The atomic for the NEXT item is normally issued when the current one is taken (its round trip and
	// the G-buffer prefetch overlap the current block's shading).  After a block with a long light list
	// the warp stops reserving ahead: a reserved block is a block no idle warp can take, and a dense
	// block can take 100 us.
	unsigned pend_got = 0;
	bool pending = false, dense_mode = false;
	auto issue_grab = [&]() {
		if (lane == 0)
			pend_got = atomicAdd(&a.queue->next_block, 1u);
		pending = true;
	};
	struct Item
	{
		int x, y;       // this lane's pixel pair
		int px0, py0;   // first pixel of the block
		int strip;
	};
	auto fetch_item = [&](Item &it) -> bool {
		if (!pending)
			issue_grab();
		const unsigned item = __shfl_sync(0xffffffffu, pend_got, 0);
		pending = false;
		if (item >= total)
			return false;
		// no reservation ahead of time near the end of the queue or in dense regions
		if (!dense_mode && item + 6u * n_warps < total)
			issue_grab();
#ifdef GRB_LIGHTING_DEBUG
		if (lane == 0)
		{
			const unsigned wid = blockIdx.x * kPWarps + warp;
			g_dbg_warp_items[wid]++;
			g_dbg_warp_last[wid][g_dbg_warp_items[wid] & 7u] = make_uint2(item, (uint32_t)(globaltimer_ns() - g_dbg_t0));
		}
#endif
		const unsigned row = item / (unsigned)a.blocks_x;
		const unsigned i = item - row * (unsigned)a.blocks_x;
		it.strip = scheduled ? (int)s_order[row] : (int)row;
		it.px0 = (int)i * 16;
		it.py0 = strips.first_row(p, it.strip);
		it.x = it.px0 + 2 * (lane & 7);
		it.y = it.py0 + (lane >> 3);
		return true;
	};
	// The G-buffer words of the NEXT block are copied asynchronously (cp.async, no registers held)
	// into this lane's 48-byte slot while the current block is shaded: the HBM round trip at the head
	// of every block otherwise leaves the warp idle for a seventh of its time.
	const uint32_t pf_slot = smem_u32(s_prefetch + (size_t)threadIdx.x * kSlotBytes);
	auto prefetch_gbuffer = [&](const Item &it) {
		const int x = it.x, y = it.y;
		if (x < p.hdr.w && y < p.y1)
		{
			asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(pf_slot), "l"(&p.depth.at(x, y)) : "memory");
			asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(pf_slot + 8u), "l"(&p.albedo.at(x, y)) : "memory");
			asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(pf_slot + 16u), "l"(&p.normal.at(x, y)) : "memory");
			asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(pf_slot + 24u), "l"(&p.emissive.at(x, y)) : "memory");
			asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(pf_slot + 32u), "l"(&p.pbr.at(x, y)) : "memory");
		}
		asm volatile("cp.async.commit_group;" ::: "memory");
	};

#ifdef GRB_LIGHTING_DEBUG
	if (threadIdx.x == 0 && blockIdx.x == 0)
		g_dbg_t0 = globaltimer_ns();
	const unsigned long long s_t0 = globaltimer_ns();
#endif
	Item nxt;
	bool have = fetch_item(nxt);
	if (have)
		prefetch_gbuffer(nxt);
	while (have)
	{
		const long long t_begin = clock64();
		const Item cur = nxt;
		const int cur_by = cur.strip;
		const int x = cur.x, y = cur.y;
		const bool inside = x < p.hdr.w && y < p.y1;

		// ---- G-buffer words (prefetched) and per-pixel invariants ----
		float2 depth = make_float2(0.f, 0.f);
		uint2 a8 = make_uint2(0u, 0u), n10 = make_uint2(0u, 0u), em = make_uint2(0u, 0u);
		uint32_t mr2 = 0u;
		asm volatile("cp.async.wait_group 0;" ::: "memory");
		if (inside)
		{
			const unsigned char *slot = s_prefetch + (size_t)threadIdx.x * kSlotBytes;
			depth = *reinterpret_cast<const float2 *>(slot);
			a8 = *reinterpret_cast<const uint2 *>(slot + 8);
			n10 = *reinterpret_cast<const uint2 *>(slot + 16);
			em = *reinterpret_cast<const uint2 *>(slot + 24);
			mr2 = *reinterpret_cast<const uint32_t *>(slot + 32);
		}
		// the slot is free again: start on the next block's words -- unless the warp is in a dense region,
		// where the next item is only taken once this block is done (see fetch_item)
		const bool deferred = dense_mode;
		if (!deferred)
		{
			have = fetch_item(nxt);
			if (have)
				prefetch_gbuffer(nxt);
		}
		auto take_deferred = [&]() {
			if (deferred)
			{
				have = fetch_item(nxt);
				if (have)
					prefetch_gbuffer(nxt);
			}
		};

		const PixelSetup A = setup_pixel(p, s_srgb, x, y, inside, depth.x, a8.x, n10.x, mr2 & 0xffffu, em.x);
		const PixelSetup B = setup_pixel(p, s_srgb, x + 1, y, inside, depth.y, a8.y, n10.y, mr2 >> 16, em.y);
		if (!__any_sync(0xffffffffu, A.lit || B.lit))
		{
			// sky block: the attachment value is carried through
			if (inside && p.emissive.p != p.hdr.p)
				*reinterpret_cast<uint2 *>(&p.hdr.at(x, y)) = em;
			take_deferred();
			continue;
		}
		SurfaceP s;
		s.npx = make_float2(-A.pos.x, -B.pos.x); s.npy = make_float2(-A.pos.y, -B.pos.y); s.npz = make_float2(-A.pos.z, -B.pos.z);
		s.Nx = make_float2(A.N.x, B.N.x); s.Ny = make_float2(A.N.y, B.N.y); s.Nz = make_float2(A.N.z, B.N.z);
		s.Vx = make_float2(A.V.x, B.V.x); s.Vy = make_float2(A.V.y, B.V.y); s.Vz = make_float2(A.V.z, B.V.z);
		s.m2m1 = make_float2(A.m2m1, B.m2m1); s.cgd = make_float2(A.cgd, B.cgd);
		s.omk = make_float2(A.omk, B.omk); s.k = make_float2(A.k, B.k); s.Vk = make_float2(A.Vk, B.Vk);
		s.nNoVr = make_float2(-A.NoVr, -B.NoVr);
		// per channel: result = Ad * S1 + F0 * S2 + S3 with Ad = dk (1 - F0)
		const f2 F0x = make_float2(A.F0.x, B.F0.x), F0y = make_float2(A.F0.y, B.F0.y), F0z = make_float2(A.F0.z, B.F0.z);
		const f2 Adx = make_float2(A.dk.x * (1.0f - A.F0.x), B.dk.x * (1.0f - B.F0.x));
		const f2 Ady = make_float2(A.dk.y * (1.0f - A.F0.y), B.dk.y * (1.0f - B.F0.y));
		const f2 Adz = make_float2(A.dk.z * (1.0f - A.F0.z), B.dk.z * (1.0f - B.F0.z));

		// ---- draw 1: directional.frag (LIGHTING_NO_AMBIENT, no shadows, VOLUMETRIC_DIFFUSE_FALLBACK) ----
		uint32_t dstA = A.dst, dstB = B.dst;
		{
			f2 ta, tga, tgb;
			shade_terms(s, add2(s.Vx, mk2(p.dir_dir.x)), add2(s.Vy, mk2(p.dir_dir.y)), add2(s.Vz, mk2(p.dir_dir.z)), mk2(1.0f), ta, tga, tgb);
			const f2 rx = fma2(Adx, ta, fma2(F0x, tga, tgb)), ry = fma2(Ady, ta, fma2(F0y, tga, tgb)), rz = fma2(Adz, ta, fma2(F0z, tga, tgb));
			if (A.lit)
			{
				float3 e = unpack_r11g11b10(dstA);
				dstA = pack_r11g11b10(e.x + p.dir_color.x * rx.x + A.base_color.x * 0.05f, e.y + p.dir_color.y * ry.x + A.base_color.y * 0.05f,
				                      e.z + p.dir_color.z * rz.x + A.base_color.z * 0.05f);
			}
			if (B.lit)
			{
				float3 e = unpack_r11g11b10(dstB);
				dstB = pack_r11g11b10(e.x + p.dir_color.x * rx.y + B.base_color.x * 0.05f, e.y + p.dir_color.y * ry.y + B.base_color.y * 0.05f,
				                      e.z + p.dir_color.z * rz.y + B.base_color.z * 0.05f);
			}
		}

		// ---- draw 2, step 1: candidate words.  Lane j owns words j, j + 32, j + 64, j + 96. ----
		// The block's cluster tiles follow from its pixel rectangle alone (the per-pixel tile index is a
		// monotone function of x and of y), so the tile loop is warp-uniform: no votes, no shuffles.
		// Every tile's bitmask row is cut to the hull of the Z-slice light ranges of the block's lit
		// pixels -- a superset of each pixel's own (tile, slice) mask; the box test below removes what
		// lies between two depth layers or in a neighbouring tile only.
		uint32_t cand0 = 0u, cand1 = 0u, cand2 = 0u, cand3 = 0u;
		{
			const unsigned lo = __reduce_min_sync(0xffffffffu, min(A.lit ? A.rx : 0xffffffffu, B.lit ? B.rx : 0xffffffffu));
			const unsigned hi = __reduce_max_sync(0xffffffffu, max(A.lit ? A.ry : 0u, B.lit ? B.ry : 0u));
			if (lo <= hi) // otherwise empty slices only: (0xffffffff, 0)
			{
				const int px0 = cur.px0, py0 = cur.py0; // the block's first pixel
				const int px1 = min(px0 + 15, p.hdr.w - 1), py1 = min(py0 + 3, p.y1 - 1);
				const int tx0 = cluster_tile_x(p, px0), tx1 = cluster_tile_x(p, px1), ty0 = cluster_tile_y(p, py0), ty1 = cluster_tile_y(p, py1);
				// cluster_mask_range (clusterer_bindless_buffers.h:17-27) for a warp-uniform range: only the
				// first and the last word of [lo, hi] are cut
				const unsigned wlo = lo >> 5, whi_raw = hi >> 5, whi = min(whi_raw, (unsigned)p.n32 - 1u);
				const uint32_t cut_lo = 0xffffffffu << (lo & 31u), cut_hi = 0xffffffffu >> (31u - (hi & 31u));
				auto cut = [&](unsigned j) -> uint32_t {
					return (j < wlo || j > whi) ? 0u : ((j == wlo ? cut_lo : 0xffffffffu) & (j == whi_raw ? cut_hi : 0xffffffffu));
				};
				const uint32_t m0 = cut((unsigned)lane), m1 = cut((unsigned)lane + 32u), m2 = cut((unsigned)lane + 64u), m3 = cut((unsigned)lane + 96u);
				for (int ty = ty0; ty <= ty1; ty++)
					for (int tx = tx0; tx <= tx1; tx++)
					{
						const uint32_t *row = p.bitmask + (size_t)(ty * p.res_x + tx) * (size_t)p.n32;
						if (m0) cand0 |= __ldg(row + lane) & m0;
						if (m1) cand1 |= __ldg(row + lane + 32) & m1;
						if (m2) cand2 |= __ldg(row + lane + 64) & m2;
						if (m3) cand3 |= __ldg(row + lane + 96) & m3;
					}
			}
		}

		// world-space bounding box of the block's lit pixels (float warp reductions)
		float bmin_x, bmin_y, bmin_z, bmax_x, bmax_y, bmax_z;
		{
			const float kBig = 3.0e38f;
			const float ax = A.lit ? A.pos.x : kBig, ay = A.lit ? A.pos.y : kBig, az = A.lit ? A.pos.z : kBig;
			const float bxx = B.lit ? B.pos.x : kBig, byy = B.lit ? B.pos.y : kBig, bzz = B.lit ? B.pos.z : kBig;
			bmin_x = warp_min_f32(fminf(ax, bxx)); bmin_y = warp_min_f32(fminf(ay, byy)); bmin_z = warp_min_f32(fminf(az, bzz));
			bmax_x = warp_max_f32(fmaxf(A.lit ? A.pos.x : -kBig, B.lit ? B.pos.x : -kBig));
			bmax_y = warp_max_f32(fmaxf(A.lit ? A.pos.y : -kBig, B.lit ? B.pos.y : -kBig));
			bmax_z = warp_max_f32(fmaxf(A.lit ? A.pos.z : -kBig, B.lit ? B.pos.z : -kBig));
		}
		if (!table_ready)
		{
			// the light table (bulk copy issued at kernel start) must have landed before its first use
			uint32_t done = 0;
			while (!done)
				asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], 0; selp.u32 %0, 1, 0, q; }" : "=r"(done) : "r"(bar) : "memory");
			table_ready = true;
		}

		// ---- draw 2, steps 2 + 3: compact the candidates that touch the box into the list, shade the list ----
		f2 S1x = mk2(0.f), S1y = mk2(0.f), S1z = mk2(0.f), S2x = mk2(0.f), S2y = mk2(0.f), S2z = mk2(0.f), S3x = mk2(0.f), S3y = mk2(0.f), S3z = mk2(0.f);
		int k = 0;
		unsigned nz = __ballot_sync(0xffffffffu, cand0 != 0u);
		bool more = true;
		int list_total = 0;
		while (more)
		{
			int count = 0;
			while (count <= kListCap - 32)
			{
				while (nz == 0u && k < 3)
				{
					k++;
					nz = __ballot_sync(0xffffffffu, (k == 1 ? cand1 : (k == 2 ? cand2 : cand3)) != 0u);
				}
				if (nz == 0u)
				{
					more = false;
					break;
				}
				const int j = __ffs(nz) - 1;
				nz &= nz - 1u;
				const uint32_t mine = k == 0 ? cand0 : (k == 1 ? cand1 : (k == 2 ? cand2 : cand3));
				const uint32_t word = __shfl_sync(0xffffffffu, mine, j);
				const unsigned widx = (unsigned)(j + 32 * k);
				const unsigned li = widx * 32u + (unsigned)lane;
				bool pass = false;
				if ((word >> lane) & 1u)
				{
					const float4 l1 = s_rec[3u * li + 1u];
					const float inv_r = s_rec[3u * li + 2u].w;
					const float dx = fmaxf(fmaxf(bmin_x - l1.x, l1.x - bmax_x), 0.0f);
					const float dy = fmaxf(fmaxf(bmin_y - l1.y, l1.y - bmax_y), 0.0f);
					const float dz = fmaxf(fmaxf(bmin_z - l1.z, l1.z - bmax_z), 0.0f);
					pass = (dx * dx + dy * dy + dz * dz) * (inv_r * inv_r) < 1.0005f;
				}
				const unsigned m = __ballot_sync(0xffffffffu, pass);
				if (pass)
				{
					const unsigned is_spot = ((__ldg(&p.type_mask[widx]) >> lane) & 1u) ^ 1u;
					list[count + __popc(m & lt_mask)] = (uint16_t)(li | (is_spot << 15));
				}
				count += __popc(m);
			}
			if (count == 0)
				break;
			list_total += count;
			if (lane == 0)
				list[count] = (uint16_t)dummy_entry; // pads an odd batch
			__syncwarp();
			if (!kPairLights)
			{
				// one light per iteration: a third fewer live registers, which buys four more warps per SM
				for (int e = 0; e < count; e++)
				{
					const unsigned ent = list[e];
					const unsigned i0 = ent & 0x7fffu;
					const float4 a0 = s_rec[3u * i0], a1 = s_rec[3u * i0 + 1u], a2 = s_rec[3u * i0 + 2u];
					f2 ta, tga, tgb;
					if (ent & 0x8000u)
						light_terms<true>(s, a0, a1, a2, true, ta, tga, tgb);
					else
						light_terms<false>(s, a0, a1, a2, false, ta, tga, tgb);
					S1x = fma2(mk2(a0.x), ta, S1x); S1y = fma2(mk2(a0.y), ta, S1y); S1z = fma2(mk2(a0.z), ta, S1z);
					S2x = fma2(mk2(a0.x), tga, S2x); S2y = fma2(mk2(a0.y), tga, S2y); S2z = fma2(mk2(a0.z), tga, S2z);
					S3x = fma2(mk2(a0.x), tgb, S3x); S3y = fma2(mk2(a0.y), tgb, S3y); S3z = fma2(mk2(a0.z), tgb, S3z);
				}
			}
			uint32_t two_next = *reinterpret_cast<const uint32_t *>(list);
			for (int e = 0; kPairLights && e < count; e += 2)
			{
				const uint32_t two = two_next;
				two_next = *reinterpret_cast<const uint32_t *>(list + e + 2); // in bounds: the list has room for kListCap + 2 entries
				const unsigned i0 = two & 0x7fffu, i1 = (two >> 16) & 0x7fffu;
				const bool spot0 = (two & 0x8000u) != 0u, spot1 = (two & 0x80000000u) != 0u;
				const float4 a0 = s_rec[3u * i0], a1 = s_rec[3u * i0 + 1u], a2 = s_rec[3u * i0 + 2u];
				const float4 b0 = s_rec[3u * i1], b1 = s_rec[3u * i1 + 1u], b2 = s_rec[3u * i1 + 2u];
				f2 ta, tga, tgb, ua, uga, ugb;
				if (two & 0x80008000u)
				{
					light_terms<true>(s, a0, a1, a2, spot0, ta, tga, tgb);
					light_terms<true>(s, b0, b1, b2, spot1, ua, uga, ugb);
				}
				else
				{
					light_terms<false>(s, a0, a1, a2, false, ta, tga, tgb);
					light_terms<false>(s, b0, b1, b2, false, ua, uga, ugb);
				}
				S1x = fma2(mk2(a0.x), ta, S1x); S1y = fma2(mk2(a0.y), ta, S1y); S1z = fma2(mk2(a0.z), ta, S1z);
				S2x = fma2(mk2(a0.x), tga, S2x); S2y = fma2(mk2(a0.y), tga, S2y); S2z = fma2(mk2(a0.z), tga, S2z);
				S3x = fma2(mk2(a0.x), tgb, S3x); S3y = fma2(mk2(a0.y), tgb, S3y); S3z = fma2(mk2(a0.z), tgb, S3z);
				S1x = fma2(mk2(b0.x), ua, S1x); S1y = fma2(mk2(b0.y), ua, S1y); S1z = fma2(mk2(b0.z), ua, S1z);
				S2x = fma2(mk2(b0.x), uga, S2x); S2y = fma2(mk2(b0.y), uga, S2y); S2z = fma2(mk2(b0.z), uga, S2z);
				S3x = fma2(mk2(b0.x), ugb, S3x); S3y = fma2(mk2(b0.y), ugb, S3y); S3z = fma2(mk2(b0.z), ugb, S3z);
			}
			__syncwarp();
		}

		if (inside)
		{
			const f2 rx = fma2(Adx, S1x, fma2(F0x, S2x, S3x)), ry = fma2(Ady, S1y, fma2(F0y, S2y, S3y)), rz = fma2(Adz, S1z, fma2(F0z, S2z, S3z));
			uint2 out = make_uint2(dstA, dstB);
			if (A.lit)
			{
				float3 e = unpack_r11g11b10(dstA);
				out.x = pack_r11g11b10(e.x + rx.x, e.y + ry.x, e.z + rz.x);
			}
			if (B.lit)
			{
				float3 e = unpack_r11g11b10(dstB);
				out.y = pack_r11g11b10(e.x + rx.y, e.y + ry.y, e.z + rz.y);
			}
			if (A.lit || B.lit || p.emissive.p != p.hdr.p)
				*reinterpret_cast<uint2 *>(&p.hdr.at(x, y)) = out;
		}
		if (a.schedule && lane == 0)
			atomicMax(&a.schedule[4 + cur_by], (uint32_t)((clock64() - t_begin) >> 5)); // key = the strip's most expensive block
		dense_mode = list_total > 96;
		take_deferred();
#ifdef GRB_LIGHTING_DEBUG
		if (lane == 0)
		{
			const int bi = cur_by * a.blocks_x + (cur.px0 >> 4);
			if (bi < kDbgBlocks)
				g_dbg_block[bi] = make_uint2((uint32_t)(clock64() - t_begin), (uint32_t)(globaltimer_ns() - s_t0));
		}
#endif
	}

#ifdef GRB_LIGHTING_DEBUG
	if (lane == 0)
		g_dbg_warp_end[blockIdx.x * kPWarps + warp] = make_uint2((uint32_t)(s_t0 & 0xffffffffu), (uint32_t)(globaltimer_ns() - s_t0));
#endif
	if (!table_ready)
	{
		// never leave with the bulk copy still in flight towards this CTA's shared memory
		uint32_t done = 0;
		while (!done)
			asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], 0; selp.u32 %0, 1, 0, q; }" : "=r"(done) : "r"(bar) : "memory");
	}
	__syncthreads();
	// The last CTA to finish re-arms the queue slot for its next launch and turns this launch's row
	// costs into the next launch's schedule (rank sort; the light table's shared memory is free now).
	uint32_t *s_flag = reinterpret_cast<uint32_t *>(s_bar + 1);
	if (threadIdx.x == 0)
	{
		__threadfence();
		const bool last = atomicAdd(&a.queue->ctas_done, 1u) == gridDim.x - 1u;
		if (last)
		{
			a.queue->next_block = 0u;
			a.queue->ctas_done = 0u;
			__threadfence();
		}
		*s_flag = last ? 1u : 0u;
	}
	__syncthreads();
	if (*s_flag && a.schedule && a.blocks_y <= kMaxOrderRows && (size_t)a.blocks_y * 4u <= (size_t)rec_total)
	{
		uint32_t *s_cost = reinterpret_cast<uint32_t *>(smem_raw);
		volatile uint32_t *cost = a.schedule + 4;
		for (int i = threadIdx.x; i < a.blocks_y; i += blockDim.x)
			s_cost[i] = cost[i];
		__syncthreads();
		for (int i = threadIdx.x; i < a.blocks_y; i += blockDim.x)
		{
			const uint32_t mine = s_cost[i];
			int rank = 0;
			for (int j = 0; j < a.blocks_y; j++)
			{
				const uint32_t c = s_cost[j];
				rank += (c > mine || (c == mine && j < i)) ? 1 : 0;
			}
			a.schedule[4 + a.blocks_y + rank] = (uint32_t)i;
			a.schedule[4 + i] = 0u;
		}
		__syncthreads();
		if (threadIdx.x == 0)
		{
			a.schedule[0] = (uint32_t)a.blocks_x;
			a.schedule[1] = (uint32_t)a.blocks_y;
			a.schedule[2] = 1u;
			__threadfence();
		}
	}
	else if (*s_flag && a.schedule)
	{
		// too many rows for the in-kernel sort: raster order next time, costs cleared
		for (int i = threadIdx.x; i < a.blocks_y; i += blockDim.x)
			a.schedule[4 + i] = 0u;
		if (threadIdx.x == 0)
			a.schedule[2] = 0u;
	}
}

// ---------------------------------------------------------------------------------------------
// Work estimate of the lighting pass per group of 4 pixel rows (one row of CTAs), in issued warp
// instructions.  The light density of a frame is far from uniform (in the bench scene 3 % of the
// rows hold over half of the light evaluations), so equal-height row bands do not split the pass
// equally between GPUs.  This kernel repeats the lighting kernel's cluster walk for the same
// 16x4 pixel blocks -- position, (tile, Z slice), word range, union of the lanes' masks, radius
// test -- without shading, and charges each step what the shading kernel's SASS spends on it.
constexpr uint32_t kCostSetup = 700u;   // per warp: G-buffer decode, position, BRDF invariants, directional light, stores
constexpr uint32_t kCostWord = 45u;     // per 32-light word of the Z range: two mask loads, range masks, warp OR
constexpr uint32_t kCostUnion = 29u;    // per light in the warp's union: record load, distance, radius vote
constexpr uint32_t kCostEvaluate = 89u; // per light that reaches a pixel of the block: falloff, cone, BRDF, accumulate

__global__ void __launch_bounds__(32 * kWarpsPerCta) lighting_cost_kernel(const LightingParams p, uint32_t *__restrict__ cost)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int x = ((blockIdx.x * kWarpsPerCta + warp) * 8 + (lane & 7)) * 2;
	const int y = p.y0 + blockIdx.y * 4 + (lane >> 3);
	if (__all_sync(0xffffffffu, x >= p.depth.w || y >= p.y1))
		return;
	float3 pos[2];
	uint32_t rx[2] = { 0xffffffffu, 0xffffffffu }, ry[2] = { 0u, 0u };
	int base[2] = { 0, 0 };
	bool lit[2] = { false, false };
#pragma unroll
	for (int k = 0; k < 2; k++)
	{
		pos[k] = make_float3(0.f, 0.f, 0.f);
		if (x + k < p.depth.w && y < p.y1)
		{
			const float depth = __ldg(&p.depth.at(x + k, y));
			if (depth != 0.0f)
			{
				int tile_index, z_index;
				pos[k] = reconstruct_position_and_cluster(p, x + k, y, depth, tile_index, z_index);
				base[k] = tile_index * p.n32;
				const uint2 zr = __ldg(&p.cluster_range[z_index]);
				rx[k] = zr.x;
				ry[k] = zr.y;
				lit[k] = true;
			}
		}
	}
	const uint32_t lo0 = rx[0] >> 5, hi0 = ry[0] >> 5, lo1 = rx[1] >> 5, hi1 = ry[1] >> 5;
	int z_start = (int)__reduce_min_sync(0xffffffffu, min(lo0, lo1));
	int z_end = (int)__reduce_max_sync(0xffffffffu, max(lit[0] ? hi0 : 0u, lit[1] ? hi1 : 0u));
	z_end = min(z_end, p.n32 - 1);
	uint32_t total = kCostSetup;
	for (int i = z_start; i <= z_end; i++)
	{
		uint32_t own0 = 0u, own1 = 0u;
		if (lit[0] && (uint32_t)i >= lo0 && (uint32_t)i <= hi0)
			own0 = cluster_mask_range(__ldg(&p.bitmask[base[0] + i]), rx[0], ry[0], 32u * (uint32_t)i);
		if (lit[1] && (uint32_t)i >= lo1 && (uint32_t)i <= hi1)
			own1 = cluster_mask_range(__ldg(&p.bitmask[base[1] + i]), rx[1], ry[1], 32u * (uint32_t)i);
		uint32_t wmask = __reduce_or_sync(0xffffffffu, own0 | own1);
		total += kCostWord;
		while (wmask)
		{
			const int bit = __ffs(wmask) - 1;
			wmask &= wmask - 1u;
			const float4 *lp = reinterpret_cast<const float4 *>(p.lights + (i * 32 + bit));
			const float4 l1 = __ldg(lp + 1), l2 = __ldg(lp + 2);
			const float inv_r2 = l2.w * l2.w;
			const float3 a = make_float3(l1.x - pos[0].x, l1.y - pos[0].y, l1.z - pos[0].z);
			const float3 b = make_float3(l1.x - pos[1].x, l1.y - pos[1].y, l1.z - pos[1].z);
			const bool near = (((own0 >> bit) & 1u) && dot3(a, a) * inv_r2 < 1.0f) || (((own1 >> bit) & 1u) && dot3(b, b) * inv_r2 < 1.0f);
			total += __any_sync(0xffffffffu, near) ? (kCostUnion + kCostEvaluate) : kCostUnion;
		}
	}
	if (lane == 0)
		atomicAdd(&cost[blockIdx.y], total);
}
} // namespace

// per-device launch state of the persistent kernel (one process may drive several GPUs)
constexpr int kMaxDevices = 64;
struct DeviceInfo
{
	std::atomic<bool> ready{ false };
	int sm_count = 0, smem_max = 0;
	QueueSlot *queue = nullptr;
	std::atomic<unsigned> next_slot{ 0 };
};
static DeviceInfo g_device_info[kMaxDevices];
static std::mutex g_device_lock;

int32_t upload_srgb_lut(const float *lut256)
{
	cudaError_t err = cudaMemcpyToSymbol(g_srgb8_to_linear, lut256, 256 * sizeof(float));
	if (err != cudaSuccess)
	{
		set_last_error(cudaGetErrorString(err));
		return GRB_ERR_CUDA;
	}
	return GRB_OK;
}
} // namespace grb

using namespace grb;

#ifdef GRB_LIGHTING_DEBUG
extern "C" int32_t grb_debug_lighting_dump(void *blocks, void *warps)
{
	cudaDeviceSynchronize();
	cudaMemcpyFromSymbol(blocks, g_dbg_block, sizeof(uint2) * kDbgBlocks);
	cudaMemcpyFromSymbol(warps, g_dbg_warp_end, sizeof(uint2) * 256 * 16);
	return 0;
}
extern "C" int32_t grb_debug_lighting_dump2(void *items, void *last)
{
	cudaMemcpyFromSymbol(items, g_dbg_warp_items, sizeof(unsigned) * 256 * 16);
	cudaMemcpyFromSymbol(last, g_dbg_warp_last, sizeof(uint2) * 256 * 16 * 8);
	static unsigned zero[256 * 16];
	cudaMemcpyToSymbol(g_dbg_warp_items, zero, sizeof(zero));
	return 0;
}
#endif

extern "C" uint64_t grb_lighting_schedule_bytes(int32_t height)
{
	const uint64_t rows = (uint64_t)((height > 0 ? height : 0) + 3) / 4;
	return (4u + 2u * rows) * sizeof(uint32_t); // header, cost and order per strip
}

extern "C" int32_t grb_deferred_lighting(const GrbGBuffer *g, const GrbCamera *cam, const GrbClusterParameters *params, const GrbClusterBuffers *buf,
                                         const GrbImage *hdr, GrbRows rows, void *stream)
{
	return grb_deferred_lighting_scheduled(g, cam, params, buf, hdr, rows, nullptr, stream);
}

static int32_t launch_deferred_lighting(const GrbGBuffer *g, const GrbCamera *cam, const GrbClusterParameters *params, const GrbClusterBuffers *buf,
                                        const GrbImage *hdr, GrbRows rows, void *schedule, void *stream, bool blocks_only, const GrbLightShadows *shadows = nullptr,
                                        const GrbStripes *stripes = nullptr);

extern "C" int32_t grb_deferred_lighting_scheduled(const GrbGBuffer *g, const GrbCamera *cam, const GrbClusterParameters *params,
                                                   const GrbClusterBuffers *buf, const GrbImage *hdr, GrbRows rows, void *schedule, void *stream)
{
	return launch_deferred_lighting(g, cam, params, buf, hdr, rows, schedule, stream, false);
}

// The same pass as a plain grid of short-lived CTAs (the non-persistent pairs kernel, one CTA per 64x4 pixel
// block; the one-pixel kernel where rows are not aligned pixel pairs) instead of persistent ones.  A persistent
// CTA keeps its SM until the work queue is empty; these free their SMs as they finish.  Results are within the
// same parity bar; the two forms associate the per-light sums differently, so they are not bit-identical to
// each other.
extern "C" int32_t grb_deferred_lighting_blocks(const GrbGBuffer *g, const GrbCamera *cam, const GrbClusterParameters *params, const GrbClusterBuffers *buf,
                                                const GrbImage *hdr, GrbRows rows, void *stream)
{
	return launch_deferred_lighting(g, cam, params, buf, hdr, rows, nullptr, stream, true);
}

// Shadowed positional lights: the generic one-pixel-per-thread kernel with the comparison sampling of grb_shadow.cuh.
// (The persistent two-pixel kernel carries no shadow path yet: DESIGN.md section 8.)
extern "C" int32_t grb_deferred_lighting_shadowed(const GrbGBuffer *g, const GrbCamera *cam, const GrbClusterParameters *params, const GrbClusterBuffers *buf,
                                                  const GrbLightShadows *shadows, const GrbImage *hdr, GrbRows rows, void *stream)
{
	if (!shadows)
	{
		set_last_error("grb_deferred_lighting_shadowed: null shadows (use grb_deferred_lighting for unshadowed lights)");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (params && params->num_lights > 0 && (!shadows->transforms || !shadows->maps || shadows->resolution <= 0 || shadows->resolution > 16384))
	{
		set_last_error("grb_deferred_lighting_shadowed: transforms / maps must be device arrays of num_lights entries, resolution in 1..16384");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	return launch_deferred_lighting(g, cam, params, buf, hdr, rows, nullptr, stream, true, shadows);
}

// Lighting of a stripe set (rows [first + k period, first + k period + rows), clipped to the image): the persistent
// kernel takes the set's strips as its work items in one launch; the other forms run one launch per stripe.
extern "C" int32_t grb_deferred_lighting_stripes(const GrbGBuffer *g, const GrbCamera *cam, const GrbClusterParameters *params,
                                                 const GrbClusterBuffers *buf, const GrbLightShadows *shadows, const GrbImage *hdr, GrbStripes stripes,
                                                 void *schedule, void *stream)
{
	if (stripes.first < 0 || stripes.rows < 4 || stripes.rows % 4 != 0 || stripes.period < stripes.rows)
	{
		set_last_error("grb_deferred_lighting_stripes: stripes need first >= 0, rows a positive multiple of 4 and period >= rows");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (shadows && params && params->num_lights > 0 && (!shadows->transforms || !shadows->maps || shadows->resolution <= 0 || shadows->resolution > 16384))
	{
		set_last_error("grb_deferred_lighting_stripes: transforms / maps must be device arrays of num_lights entries, resolution in 1..16384");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	return launch_deferred_lighting(g, cam, params, buf, hdr, GrbRows{ 0, 0 }, shadows ? nullptr : schedule, stream, shadows != nullptr, shadows, &stripes);
}

// What a pixel's position and (tile, Z slice) follow from: the camera, the cluster grid and the image size.
static void set_cluster_geometry(LightingParams &p, const GrbCamera *cam, const GrbClusterParameters *params, int w, int h, GrbRows rows)
{
	for (int i = 0; i < 16; i++)
		p.ivp[i] = cam->inv_view_projection[i];
	p.cbase = make_float3(params->camera_base[0], params->camera_base[1], params->camera_base[2]);
	p.cfront = make_float3(params->camera_front[0], params->camera_front[1], params->camera_front[2]);
	p.xy_scale = make_float2(params->xy_scale[0], params->xy_scale[1]);
	p.res_x = params->resolution_xy[0];
	p.res_y = params->resolution_xy[1];
	p.n32 = params->num_lights_32;
	p.z_max_index = params->z_max_index;
	p.z_scale = params->z_scale;
	p.inv_res_x = 1.0f / (float)w; // renderer.cpp:1101-1102,1120
	p.inv_res_y = 1.0f / (float)h;
	p.y0 = rows.y0;
	p.y1 = rows.y1;
}

static int32_t launch_deferred_lighting(const GrbGBuffer *g, const GrbCamera *cam, const GrbClusterParameters *params, const GrbClusterBuffers *buf,
                                        const GrbImage *hdr, GrbRows rows, void *schedule, void *stream, bool blocks_only, const GrbLightShadows *shadows,
                                        const GrbStripes *stripes)
{
	if (!g || !cam || !params || !buf || !hdr)
	{
		set_last_error("grb_deferred_lighting: null argument");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	const bool hdr16 = image_ok(hdr, GRB_FORMAT_R16G16B16A16_SFLOAT, 8); // "renderTargetFp16"
	if (!image_ok(&g->albedo, GRB_FORMAT_R8G8B8A8_SRGB, 4) || !image_ok(&g->normal, GRB_FORMAT_A2B10G10R10_UNORM_PACK32, 4) ||
	    !image_ok(&g->pbr, GRB_FORMAT_R8G8_UNORM, 2) || !image_ok(&g->depth, GRB_FORMAT_D32_SFLOAT, 4) ||
	    (!hdr16 && !image_ok(hdr, GRB_FORMAT_B10G11R11_UFLOAT_PACK32, 4)))
	{
		set_last_error("grb_deferred_lighting: G-buffer must be R8G8B8A8_SRGB / A2B10G10R10_UNORM / R8G8_UNORM / D32_SFLOAT, hdr B10G11R11_UFLOAT or R16G16B16A16_SFLOAT");
		return GRB_ERR_UNSUPPORTED_FORMAT;
	}
	const int w = hdr->width, h = hdr->height;
	if (g->albedo.width != w || g->albedo.height != h || g->normal.width != w || g->normal.height != h || g->pbr.width != w || g->pbr.height != h ||
	    g->depth.width != w || g->depth.height != h)
	{
		set_last_error("grb_deferred_lighting: attachment sizes differ");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (params->num_lights > 0 && (!buf->lights || !buf->type_mask || !buf->bitmask))
	{
		set_last_error("grb_deferred_lighting: null cluster buffer");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (!buf->cluster_range)
	{
		set_last_error("grb_deferred_lighting: null cluster_range");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (reinterpret_cast<uintptr_t>(buf->lights) % 16 != 0)
	{
		// every form reads the records as float4 (and the persistent one bulk-copies them)
		set_last_error("grb_deferred_lighting: lights must be 16-byte aligned");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	rows = stripes ? GrbRows{ stripes->first, h } : full_rows(rows, h);
	if (rows.y1 <= rows.y0)
		return GRB_OK;

	LightingParams p;
	p.albedo = view_of<const uint32_t>(&g->albedo);
	p.normal = view_of<const uint32_t>(&g->normal);
	p.pbr = view_of<const uint16_t>(&g->pbr);
	p.depth = view_of<const float>(&g->depth);
	p.hdr = view_of<uint32_t>(hdr);
	p.hdr16 = view_of<uint2>(hdr);
	if (g->emissive.data)
	{
		if (!image_ok(&g->emissive, hdr->format, hdr16 ? 8 : 4) || g->emissive.width != w || g->emissive.height != h)
		{
			set_last_error("grb_deferred_lighting: emissive must have hdr's format (B10G11R11_UFLOAT or R16G16B16A16_SFLOAT) and the G-buffer's size");
			return GRB_ERR_UNSUPPORTED_FORMAT;
		}
		p.emissive = view_of<const uint32_t>(&g->emissive);
		p.emissive16 = view_of<const uint2>(&g->emissive);
	}
	else
	{
		p.emissive = view_of<const uint32_t>(hdr);
		p.emissive16 = view_of<const uint2>(hdr);
	}
	set_cluster_geometry(p, cam, params, w, h, rows);
	p.camera_pos = make_float3(cam->camera_position[0], cam->camera_position[1], cam->camera_position[2]);
	p.dir_color = make_float3(g->directional_color[0], g->directional_color[1], g->directional_color[2]);
	p.dir_dir = make_float3(g->directional_direction[0], g->directional_direction[1], g->directional_direction[2]);
	p.lights = buf->lights;
	p.type_mask = buf->type_mask;
	p.bitmask = buf->bitmask;
	p.cluster_range = reinterpret_cast<const uint2 *>(buf->cluster_range);
	p.shadow_transforms = shadows ? shadows->transforms : nullptr;
	p.shadow_maps = shadows ? reinterpret_cast<const uint16_t *const *>(shadows->maps) : nullptr;
	p.shadow_res = shadows ? shadows->resolution : 0;
	p.shadow_pcf_wide = shadows ? shadows->pcf_wide : 0;

	// two pixels per thread (packed fp32) whenever rows can be addressed as aligned pixel pairs
	static const bool force_1px = getenv("GRB_LIGHTING_1PX") != nullptr;
	auto aligned8 = [](const void *ptr, int pitch_bytes) { return (reinterpret_cast<uintptr_t>(ptr) % 8) == 0 && (pitch_bytes % 8) == 0; };
	const bool pairs = !shadows && !hdr16 && !force_1px && (w % 2) == 0 && aligned8(g->albedo.data, g->albedo.row_pitch) && aligned8(g->normal.data, g->normal.row_pitch) &&
	                   aligned8(g->depth.data, g->depth.row_pitch) && (reinterpret_cast<uintptr_t>(g->pbr.data) % 4) == 0 && (g->pbr.row_pitch % 4) == 0 &&
	                   aligned8(hdr->data, hdr->row_pitch) && (!g->emissive.data || aligned8(g->emissive.data, g->emissive.row_pitch));
	static const bool force_v2 = getenv("GRB_LIGHTING_V2") != nullptr;
	if (pairs && !force_v2 && !blocks_only && params->num_lights <= 4096 && params->num_lights_32 <= 128)
	{
		// persistent kernel: one CTA per SM, light table in shared memory
		int device = 0;
		cudaError_t err = cudaGetDevice(&device);
		if (err != cudaSuccess || device < 0 || device >= kMaxDevices)
		{
			set_last_error("grb_deferred_lighting: cudaGetDevice failed");
			return GRB_ERR_CUDA;
		}
		DeviceInfo &di = g_device_info[device];
		if (!di.ready.load(std::memory_order_acquire))
		{
			std::lock_guard<std::mutex> hold(g_device_lock);
			if (!di.ready.load(std::memory_order_relaxed))
			{
				int sms = 0, smem_max = 0;
				err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
				if (err == cudaSuccess)
					err = cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
				if (err == cudaSuccess)
					err = cudaFuncSetAttribute(deferred_lighting_persistent_kernel<BandStrips>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
				if (err == cudaSuccess)
					err = cudaFuncSetAttribute(deferred_lighting_persistent_kernel<StripeSetStrips>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
				void *q = nullptr;
				if (err == cudaSuccess)
					err = cudaGetSymbolAddress(&q, g_light_queue);
				if (err != cudaSuccess)
				{
					set_last_error(cudaGetErrorString(err));
					return GRB_ERR_CUDA;
				}
				di.sm_count = sms;
				di.smem_max = smem_max;
				di.queue = static_cast<QueueSlot *>(q);
				di.ready.store(true, std::memory_order_release);
			}
		}
		PersistentArgs a;
		a.blocks_x = (w + 15) / 16;
		a.blocks_y = (rows.y1 - rows.y0 + 3) / 4;
		StripeSetStrips strips = {};
		if (stripes)
		{
			// every stripe but the last that starts inside the image is whole
			const int spp = stripes->rows / 4, count = (h - stripes->first + stripes->period - 1) / stripes->period;
			const int last_rows = std::min(stripes->rows, h - (stripes->first + (count - 1) * stripes->period));
			strips = StripeSetStrips{ stripes->first, spp, stripes->period };
			a.blocks_y = (count - 1) * spp + (last_rows + 3) / 4;
		}
		a.total_items = a.blocks_x * a.blocks_y;
		a.schedule = static_cast<uint32_t *>(schedule);
		a.n_lights = params->num_lights;
		a.rec_bytes = (unsigned)params->num_lights * 48u;
		a.queue = di.queue + (di.next_slot.fetch_add(1u, std::memory_order_relaxed) % 64u);
		const size_t smem = (size_t)a.rec_bytes + 48u + 1024u + ((kPWarps * (kListCap + 2) * 2u + 15u) & ~15u) + 32u * kPWarps * kSlotBytes + 16u + kMaxOrderRows * 2u;
		if (smem <= (size_t)di.smem_max)
		{
			const int ctas = std::min(di.sm_count, std::max(1, (a.blocks_x * a.blocks_y + kPWarps - 1) / kPWarps));
			if (stripes)
				deferred_lighting_persistent_kernel<<<ctas, 32 * kPWarps, smem, as_stream(stream)>>>(p, a, strips);
			else
				deferred_lighting_persistent_kernel<<<ctas, 32 * kPWarps, smem, as_stream(stream)>>>(p, a, BandStrips{});
			return check_launch("grb_deferred_lighting");
		}
	}
	auto launch_rows = [&](int y0, int y1) {
		p.y0 = y0;
		p.y1 = y1;
		if (pairs)
		{
			dim3 grid2((w / 2 + 8 * kWarpsPerCta - 1) / (8 * kWarpsPerCta), (y1 - y0 + 3) / 4, 1);
			deferred_lighting2_kernel<<<grid2, 32 * kWarpsPerCta, 0, as_stream(stream)>>>(p);
			return;
		}
		dim3 grid((w + 8 * kWarpsPerCta - 1) / (8 * kWarpsPerCta), (y1 - y0 + 3) / 4, 1);
		if (hdr16 && shadows)
			deferred_lighting_kernel<true, true><<<grid, 32 * kWarpsPerCta, 0, as_stream(stream)>>>(p);
		else if (hdr16)
			deferred_lighting_kernel<false, true><<<grid, 32 * kWarpsPerCta, 0, as_stream(stream)>>>(p);
		else if (shadows)
			deferred_lighting_kernel<true><<<grid, 32 * kWarpsPerCta, 0, as_stream(stream)>>>(p);
		else
			deferred_lighting_kernel<false><<<grid, 32 * kWarpsPerCta, 0, as_stream(stream)>>>(p);
	};
	if (!stripes)
		launch_rows(rows.y0, rows.y1);
	else // the forms the persistent kernel does not serve: one launch per stripe
		for (int y = stripes->first; y < h; y += stripes->period)
			launch_rows(y, std::min(y + stripes->rows, h));
	return check_launch("grb_deferred_lighting");
}

extern "C" int32_t grb_debug_cluster_indices(const GrbImage *depth, const GrbCamera *cam, const GrbClusterParameters *params, int32_t *out_tile,
                                             int32_t *out_z, GrbRows rows, void *stream)
{
	if (!image_ok(depth, GRB_FORMAT_D32_SFLOAT, 4) || !cam || !params || !out_tile || !out_z)
	{
		set_last_error("grb_debug_cluster_indices: bad arguments");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	rows = full_rows(rows, depth->height);
	if (rows.y1 <= rows.y0)
		return GRB_OK;
	LightingParams p{};
	p.depth = view_of<const float>(depth);
	set_cluster_geometry(p, cam, params, depth->width, depth->height, rows);
	dim3 grid((depth->width + 31) / 32, (rows.y1 - rows.y0 + 3) / 4, 1);
	cluster_indices_kernel<<<grid, 128, 0, as_stream(stream)>>>(p, out_tile, out_z);
	return check_launch("grb_debug_cluster_indices");
}

extern "C" int32_t grb_lighting_row_cost(const GrbImage *depth, const GrbCamera *cam, const GrbClusterParameters *params, const GrbClusterBuffers *buf,
                                         GrbRows rows, uint32_t *cost_per_4_rows, void *stream)
{
	if (!image_ok(depth, GRB_FORMAT_D32_SFLOAT, 4) || !cam || !params || !buf || !cost_per_4_rows)
	{
		set_last_error("grb_lighting_row_cost: bad arguments");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (!buf->cluster_range || (params->num_lights > 0 && (!buf->lights || !buf->bitmask)))
	{
		set_last_error("grb_lighting_row_cost: null cluster buffer");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (reinterpret_cast<uintptr_t>(buf->lights) % 16 != 0)
	{
		set_last_error("grb_lighting_row_cost: lights must be 16-byte aligned");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	rows = full_rows(rows, depth->height);
	if (rows.y1 <= rows.y0)
		return GRB_OK;
	const int groups = (rows.y1 - rows.y0 + 3) / 4;
	cudaError_t err = cudaMemsetAsync(cost_per_4_rows, 0, sizeof(uint32_t) * (size_t)groups, as_stream(stream));
	if (err != cudaSuccess)
	{
		set_last_error(cudaGetErrorString(err));
		return GRB_ERR_CUDA;
	}
	LightingParams p{};
	p.depth = view_of<const float>(depth);
	set_cluster_geometry(p, cam, params, depth->width, depth->height, rows);
	p.lights = buf->lights;
	p.bitmask = buf->bitmask;
	p.cluster_range = reinterpret_cast<const uint2 *>(buf->cluster_range);
	const int pairs = (depth->width + 1) / 2;
	dim3 grid((pairs + 8 * kWarpsPerCta - 1) / (8 * kWarpsPerCta), groups, 1);
	lighting_cost_kernel<<<grid, 32 * kWarpsPerCta, 0, as_stream(stream)>>>(p, cost_per_4_rows);
	return check_launch("grb_lighting_row_cost");
}
