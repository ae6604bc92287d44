/*
 * oracle_lighting.c -- TEST INFRASTRUCTURE ONLY.  Deferred lighting pass (K6 directional +
 * K5 clustered) restated from the reference GLSL.  See oracle_math.h for arithmetic rules.
 *
 * Reference: renderer/renderer.cpp:1004-1156 (DeferredLightRenderer::render_light) issues two
 * full-screen draws with additive ONE/ONE blending into "HDR-main" (which aliases the
 * emissive attachment, B10G11R11_UFLOAT), depth test NOT_EQUAL against the quad's z=0 so sky
 * pixels (depth == 0) are untouched.  Each blend is dst = quantise(src + decode(dst)).
 */
#include "oracle.h"
#include "oracle_math.h"

#define PI_GRANITE 3.1415628f /* assets/shaders/lights/pbr.h:5 (sic) */

/* pbr.h:8-26 */
static float D_GGX(float roughness, vec3 N, vec3 H)
{
	float NoH = f_clamp(v3_dot(N, H), 0.0001f, 1.0f);
	float m = roughness * roughness;
	float m2 = m * m;
	float d = (NoH * m2 - NoH) * NoH + 1.0f;
	return m2 / (PI_GRANITE * d * d);
}

/* pbr.h:28-35 */
static float G_schlick(float roughness, float NoV, float NoL)
{
	float r = roughness + 1.0f;
	float k = r * r * (1.0f / 8.0f);
	float V = NoV * (1.0f - k) + k;
	float L = NoL * (1.0f - k) + k;
	return 0.25f / f_max(V * L, 0.001f);
}

/* pbr.h:44-47: mix(F0, vec3(1.0), pow(1.0 - HoV, 5.0)) */
static vec3 fresnel(vec3 F0, float HoV)
{
	float t = powf(1.0f - HoV, 5.0f);
	return v3(f_mix(F0.x, 1.0f, t), f_mix(F0.y, 1.0f, t), f_mix(F0.z, 1.0f, t));
}

/* pbr.h:54-57 */
static vec3 compute_F0(vec3 base_color, float metallic)
{
	return v3(f_mix(0.04f, base_color.x, metallic), f_mix(0.04f, base_color.y, metallic), f_mix(0.04f, base_color.z, metallic));
}

/* Shared tail of point.h:121-141 / spot.h:124-144 / lighting.h:26-46: Cook-Torrance BRDF.
 * Returns (reflected + diffuse) WITHOUT the light colour factor when prefactor == NULL,
 * otherwise follows lighting.h where light_color * NoL * shadow_term leads the products. */
static vec3 brdf_terms(vec3 base_color, vec3 N, float metallic, float material_roughness,
                       vec3 L, vec3 V, const vec3 *light_color_dir)
{
	float roughness = material_roughness * 0.75f + 0.25f;
	vec3 H = v3_normalize(v3_add(V, L));
	float NoV = f_clamp(v3_dot(N, V), 0.001f, 1.0f);
	float NoL = f_clamp(v3_dot(N, L), 0.001f, 1.0f);
	float HoV = f_clamp(v3_dot(H, V), 0.001f, 1.0f);
	vec3 F0 = compute_F0(base_color, metallic);
	vec3 F = fresnel(F0, HoV);
	/* cook_torrance_specular: specular * G * D */
	float D = D_GGX(roughness, N, H);
	float G = G_schlick(roughness, NoV, NoL);
	vec3 ct = v3_scale(v3_scale(F, G), D);
	vec3 specref, diffref;
	if (light_color_dir)
	{
		/* lighting.h:41-42: light_color * NoL * shadow_term(1.0) * X */
		vec3 lc = v3_scale(v3_scale(*light_color_dir, NoL), 1.0f);
		specref = v3_mul(lc, ct);
		diffref = v3_scale(v3_mul(lc, v3(1.0f - F.x, 1.0f - F.y, 1.0f - F.z)), 1.0f / PI_GRANITE);
	}
	else
	{
		/* point.h:136-137: NoL * cook_torrance ; NoL * (1 - F) * (1/PI) */
		specref = v3_scale(ct, NoL);
		diffref = v3_scale(v3(NoL * (1.0f - F.x), NoL * (1.0f - F.y), NoL * (1.0f - F.z)), 1.0f / PI_GRANITE);
	}
	/* diffuse_light = diffref * base_color * (1 - metallic) */
	vec3 diffuse = v3_scale(v3_mul(diffref, base_color), 1.0f - metallic);
	return v3_add(specref, diffuse);
}


/* ---------------------------------------------------------------------------------------------
 * Shadowed positional lights (POSITIONAL_LIGHTS_SHADOW, PCF; renderer.cpp:369,1126).
 *
 * The reference samples one D16_UNORM image per light (clusterer.cpp:397-407: 2-D for a spot light, a cube of
 * 6 layers for a point light, shadow_resolution^2 each) through StockSampler::LinearShadow
 * (vulkan/device.cpp:1086-1088,1118-1120,1146-1149): compare GREATER_OR_EQUAL, linear filter, clamp to edge.
 * A texture unit's comparison filtering is specified by the Vulkan specification ("Texel Input Operations /
 * Depth Compare Operation" then "Texel Filtering"), restated here in fp32:
 *   - D_ref is clamped to [0, 1] (fixed-point depth format), each of the 2 x 2 texels gives 1.0 where
 *     D_ref >= D_texel (D_texel = code / 65535), else 0.0;
 *   - the four results are blended with the bilinear weights of (u, v) = (s W - 0.5, t H - 0.5) -- the oracle's
 *     bilin_setup / bilin_mix, exact fp32 weights where hardware keeps 8 fractional bits;
 *   - a 2-D image clamps texel indices to the edge; a cube map selects the face by the major axis (ties: z over
 *     y over x) with the (s_c, t_c) table of the specification, and a footprint that leaves the face takes the
 *     texel across the edge from the adjacent face ("Cube Map Edge Handling"); at a corner, where the fourth
 *     texel does not exist, it is replaced by the average of the other three.
 * A NULL map means "this light casts no shadow" (shadow_falloff = 1, the unshadowed shaders).
 * --------------------------------------------------------------------------------------------- */
static float shadow_compare(const uint16_t *map, size_t texel, float ref)
{
	return ref >= (float)map[texel] / 65535.0f ? 1.0f : 0.0f;
}

/* textureProjLod(sampler2DShadow, clip, 0.0): pcf.h:98-99 (SHADOW_MAP_PCF_KERNEL_WIDE undefined) */
float orc_shadow_sample_2d(const uint16_t *map, int res, float clip_x, float clip_y, float clip_z, float clip_w)
{
	float s = clip_x / clip_w, t = clip_y / clip_w;
	float ref = f_clamp(clip_z / clip_w, 0.0f, 1.0f);
	if (!(ref == ref))
		ref = 0.0f;
	bilin_t b = bilin_setup(s, t, res, res);
	int x0 = b.x0 < 0 ? 0 : (b.x0 > res - 1 ? res - 1 : b.x0), x1 = b.x1 < 0 ? 0 : (b.x1 > res - 1 ? res - 1 : b.x1);
	int y0 = b.y0 < 0 ? 0 : (b.y0 > res - 1 ? res - 1 : b.y0), y1 = b.y1 < 0 ? 0 : (b.y1 > res - 1 ? res - 1 : b.y1);
	float c00 = shadow_compare(map, (size_t)y0 * res + x0, ref), c10 = shadow_compare(map, (size_t)y0 * res + x1, ref);
	float c01 = shadow_compare(map, (size_t)y1 * res + x0, ref), c11 = shadow_compare(map, (size_t)y1 * res + x1, ref);
	return bilin_mix(c00, c10, c01, c11, b.a, b.b);
}

/* SHADOW_MAP_PCF_KERNEL_WIDE (renderer.cpp:380-381, pcf.h:7-80): a 6 x 6 texel kernel from nine comparison gathers, weights
 * exp2(-0.375 d^2) (1 - d^2 / 9) per axis, normalised.  The gathers sit on texel corners (floor(uv res - 1.5) / res), so
 * their footprints are exact whatever the sampler's precision: texel (c, r) of the window = (fx - 1 + c, fy - 1 + r),
 * clamped to the edge.  Sums in the order of the shader's statements (dot and the weight sum as GLM / the macro write
 * them), so that the pin compares like with like; exp2 is libm's. */
static float pcf_wide_weight(float p)
{
	float p2 = p * p;
	return exp2f(p2 * -0.375f) * (1.0f - p2 / 9.0f);
}

float orc_shadow_sample_2d_wide(const uint16_t *map, int res, float clip_x, float clip_y, float clip_z, float clip_w)
{
	float u = clip_x / clip_w, v = clip_y / clip_w;
	float ref = f_clamp(clip_z / clip_w, 0.0f, 1.0f);
	if (!(ref == ref))
		ref = 0.0f;
	const float fres = (float)res;
	float ix = u * fres - 1.5f, iy = v * fres - 1.5f;
	float flx = floorf(ix), fly = floorf(iy);
	const float fx = ix - flx, fy = iy - fly;
	/* footprint origin of textureGather at floored / res: floor(floored / res * res - 0.5) = floored - 1.  Each texel of
	 * the window clamps to the edge on its own (the gathers' clamp to edge), so the origin itself is not clamped to the
	 * map; 8 texels outside, every texel already clamps to the same edge, so the bound only keeps the int conversion
	 * defined.  NaN coordinates: origin -1. */
	bilin_t b;
	b.x0 = (int)(flx == flx ? f_clamp(flx, -8.0f, fres + 8.0f) : 0.0f) - 1;
	b.y0 = (int)(fly == fly ? f_clamp(fly, -8.0f, fres + 8.0f) : 0.0f) - 1;
	float H[6], V[6];
	const float off[6] = { 2.0f, 1.0f, 0.0f, -1.0f, -2.0f, -3.0f };
	for (int i = 0; i < 6; i++)
	{
		H[i] = pcf_wide_weight(fx + off[i]);
		V[i] = pcf_wide_weight(fy + off[i]);
	}
	float c[6][6];
	for (int r = 0; r < 6; r++)
		for (int q = 0; q < 6; q++)
		{
			int x = b.x0 + q, y = b.y0 + r;
			x = x < 0 ? 0 : (x > res - 1 ? res - 1 : x);
			y = y < 0 ? 0 : (y > res - 1 ? res - 1 : y);
			c[r][q] = shadow_compare(map, (size_t)y * res + x, ref);
		}
	float var = 0.0f, total_w = 0.0f;
	for (int gy = 0; gy < 3; gy++)
		for (int gx = 0; gx < 3; gx++)
		{
			const int a = 2 * gx, p = 2 * gy; /* gather components: x = (a, p + 1), y = (a + 1, p + 1), z = (a + 1, p), w = (a, p) */
			const float kx = H[a] * V[p + 1], ky = H[a + 1] * V[p + 1], kz = H[a + 1] * V[p], kw = H[a] * V[p];
			var += (c[p + 1][a] * kx + c[p + 1][a + 1] * ky) + (c[p][a + 1] * kz + c[p][a] * kw);
			total_w += (kx + kz) + (ky + kw);
		}
	return var / total_w;
}

/* Texel (i, j) of cube face f, where i or j may be one step outside [0, res): the texel across that edge.
 * Worked in doubled integer coordinates on the cube of half-size `res`: a texel centre of face f is the point
 * with major-axis component +-res and in-face components 2 i + 1 - res (odd, |.| < res).  One step outside
 * gives +-(res + 1): that axis becomes the major one (+-res) and the old major axis holds the edge texel of
 * the neighbouring face, +-(res - 1).  Returns 0 at a corner (both outside). */
int orc_shadow_cube_texel(int res, int f, int i, int j, size_t *texel)
{
	int a = 2 * i + 1 - res, b = 2 * j + 1 - res; /* s_c, t_c in doubled texel units */
	int out_a = a < -res || a > res, out_b = b < -res || b > res;
	if (out_a && out_b)
		return 0;
	/* face -> direction (x, y, z): inverse of the specification's table (s_c, t_c, m_a) */
	int m = res, x, y, z;
	switch (f)
	{
	case 0: x = m; y = -b; z = -a; break;  /* +X: s_c = -z, t_c = -y */
	case 1: x = -m; y = -b; z = a; break;  /* -X: s_c = +z, t_c = -y */
	case 2: x = a; y = m; z = b; break;    /* +Y: s_c = +x, t_c = +z */
	case 3: x = a; y = -m; z = -b; break;  /* -Y: s_c = +x, t_c = -z */
	case 4: x = a; y = -b; z = m; break;   /* +Z: s_c = +x, t_c = -y */
	default: x = -a; y = -b; z = -m; break; /* -Z: s_c = -x, t_c = -y */
	}
	if (out_a || out_b)
	{
		int *v[3] = { &x, &y, &z };
		for (int k = 0; k < 3; k++)
		{
			if (*v[k] == m || *v[k] == -m)
				*v[k] = *v[k] > 0 ? res - 1 : -(res - 1); /* old major axis: edge texel of the neighbour */
			else if (*v[k] > res || *v[k] < -res)
				*v[k] = *v[k] > 0 ? res : -res; /* new major axis */
		}
		int ax = x < 0 ? -x : x, ay = y < 0 ? -y : y;
		int nf, sc, tc;
		if (ax == res) { nf = x > 0 ? 0 : 1; sc = x > 0 ? -z : z; tc = -y; }
		else if (ay == res) { nf = y > 0 ? 2 : 3; sc = x; tc = y > 0 ? z : -z; }
		else { nf = z > 0 ? 4 : 5; sc = z > 0 ? x : -x; tc = -y; }
		f = nf;
		a = sc;
		b = tc;
	}
	int ti = (a + res - 1) / 2, tj = (b + res - 1) / 2;
	*texel = ((size_t)f * res + tj) * res + ti;
	return 1;
}

/* texture(samplerCubeShadow, vec4(dir, ref)): point.h:56-71 */
float orc_shadow_sample_cube(const uint16_t *map, int res, float dx, float dy, float dz, float ref)
{
	ref = f_clamp(ref, 0.0f, 1.0f);
	if (!(ref == ref))
		ref = 0.0f;
	float ax = fabsf(dx), ay = fabsf(dy), az = fabsf(dz);
	int face;
	float sc, tc, ma;
	if (az >= ax && az >= ay) { face = dz < 0.0f ? 5 : 4; sc = dz < 0.0f ? -dx : dx; tc = -dy; ma = az; }
	else if (ay >= ax) { face = dy < 0.0f ? 3 : 2; sc = dx; tc = dy < 0.0f ? -dz : dz; ma = ay; }
	else { face = dx < 0.0f ? 1 : 0; sc = dx < 0.0f ? dz : -dz; tc = -dy; ma = ax; }
	float s = 0.5f * (sc / ma) + 0.5f, t = 0.5f * (tc / ma) + 0.5f;
	bilin_t b = bilin_setup(s, t, res, res);
	int xs[2] = { b.x0, b.x1 }, ys[2] = { b.y0, b.y1 };
	for (int k = 0; k < 2; k++)
	{
		/* a face coordinate is within [0, 1] up to rounding: the footprint is at most one texel outside */
		xs[k] = xs[k] < -1 ? -1 : (xs[k] > res ? res : xs[k]);
		ys[k] = ys[k] < -1 ? -1 : (ys[k] > res ? res : ys[k]);
	}
	float c[4];
	int have[4], n = 0;
	float sum = 0.0f;
	for (int k = 0; k < 4; k++)
	{
		size_t texel = 0;
		have[k] = orc_shadow_cube_texel(res, face, xs[k & 1], ys[k >> 1], &texel);
		c[k] = have[k] ? shadow_compare(map, texel, ref) : 0.0f;
		if (have[k]) { sum += c[k]; n++; }
	}
	if (n == 3)
		for (int k = 0; k < 4; k++)
			if (!have[k])
				c[k] = sum / 3.0f;
	return bilin_mix(c[0], c[1], c[2], c[3], b.a, b.b);
}

/* mat4 * vec4(world_pos, 1): the association of the generated reference code (GLM: (c0 x + c1 y) + (c2 z + c3 w)) */
static vec4 shadow_clip(const float *m, vec3 p)
{
	return v4((m[0] * p.x + m[4] * p.y) + (m[8] * p.z + m[12] * 1.0f), (m[1] * p.x + m[5] * p.y) + (m[9] * p.z + m[13] * 1.0f),
	          (m[2] * p.x + m[6] * p.y) + (m[10] * p.z + m[14] * 1.0f), (m[3] * p.x + m[7] * p.y) + (m[11] * p.z + m[15] * 1.0f));
}

/* the light's shadow inputs for one evaluation; map == NULL => unshadowed */
typedef struct { const float *transform; const uint16_t *map; int res; int wide; } light_shadow_t;

/* point.h:33-81 compute_point_color */
static vec3 compute_point_color(const orc_light_t *pt, vec3 world_pos, vec3 *light_dir, light_shadow_t sh)
{
	vec3 light_pos = v3(pt->position[0], pt->position[1], pt->position[2]);
	vec3 full = v3_sub(world_pos, light_pos);
	*light_dir = v3_normalize(v3_neg(full));
	float light_dist = f_max(0.1f, v3_length(full));
	float static_falloff = 1.0f - f_smoothstep(0.9f, 1.0f, light_dist * pt->inv_radius);
	if (static_falloff > 0.0f)
	{
		float shadow_falloff = 1.0f;
		if (sh.map)
		{
			/* point.h:46-49,67-71: reference depth of the cube face along the major axis */
			float max_z = f_max(f_max(fabsf(full.x), fabsf(full.y)), fabsf(full.z));
			const float *t = sh.transform; /* shadow[index][0] = (proj[2].zw, proj[3].zw), clusterer.cpp:521 */
			float ref_x = t[2] - t[0] * max_z, ref_y = t[3] - t[1] * max_z;
			shadow_falloff = orc_shadow_sample_cube(sh.map, sh.res, full.x, full.y, full.z, ref_x / ref_y);
		}
		float s = (shadow_falloff * static_falloff);
		float d2 = (light_dist * light_dist);
		/* point.color * (shadow*static) / (dist*dist): left-to-right */
		return v3(pt->color[0] * s / d2, pt->color[1] * s / d2, pt->color[2] * s / d2);
	}
	return v3(0.0f, 0.0f, 0.0f);
}

/* spot.h:34-84 compute_spot_color */
static vec3 compute_spot_color(const orc_light_t *sp, vec3 world_pos, vec3 *light_dir, light_shadow_t sh)
{
	vec3 light_pos = v3(sp->position[0], sp->position[1], sp->position[2]);
	vec3 primary = v3(sp->direction[0], sp->direction[1], sp->direction[2]);
	vec3 full = v3_sub(light_pos, world_pos);
	*light_dir = v3_normalize(full);
	float light_dist = f_max(0.1f, v3_length(full));
	float cone_angle = v3_dot(v3_normalize(v3_sub(world_pos, light_pos)), primary);
	float scale = f16_to_f32(sp->spot_scale_bias[0]); /* unpackHalf2x16 */
	float bias = f16_to_f32(sp->spot_scale_bias[1]);
	float cone_falloff = f_clamp(cone_angle * scale + bias, 0.0f, 1.0f);
	cone_falloff *= cone_falloff;
	cone_falloff *= 1.0f - f_smoothstep(0.9f, 1.0f, light_dist * sp->inv_radius);
	if (cone_falloff > 0.0f)
	{
		float shadow_falloff = 1.0f;
		if (sh.map)
		{
			/* spot.h:67-77 + pcf.h:98-99 */
			vec4 clip = shadow_clip(sh.transform, world_pos);
			shadow_falloff = sh.wide ? orc_shadow_sample_2d_wide(sh.map, sh.res, clip.x, clip.y, clip.z, clip.w)
			                         : orc_shadow_sample_2d(sh.map, sh.res, clip.x, clip.y, clip.z, clip.w);
		}
		float k = (cone_falloff * shadow_falloff) / (light_dist * light_dist);
		return v3(sp->color[0] * k, sp->color[1] * k, sp->color[2] * k);
	}
	return v3(0.0f, 0.0f, 0.0f);
}

/* point.h:103-142 / spot.h:106-145 */
static vec3 compute_positional_light(const orc_light_t *l, int is_point, vec3 base_color, vec3 N,
                                     float metallic, float roughness, vec3 world_pos, vec3 camera_pos, light_shadow_t sh)
{
	vec3 light_dir;
	vec3 color = is_point ? compute_point_color(l, world_pos, &light_dir, sh) : compute_spot_color(l, world_pos, &light_dir, sh);
	if (color.x == 0.0f && color.y == 0.0f && color.z == 0.0f)
		return v3(0.0f, 0.0f, 0.0f);
	vec3 V = v3_normalize(v3_sub(camera_pos, world_pos));
	vec3 terms = brdf_terms(base_color, N, metallic, roughness, light_dir, V, 0);
	return v3_mul(color, terms);
}

/* clusterer_bindless_buffers.h:17-27 */
static uint32_t cluster_mask_range(uint32_t mask, uint32_t rx, uint32_t ry, uint32_t start_index)
{
	uint32_t lo = start_index, hi = start_index + 32u;
	rx = rx < lo ? lo : (rx > hi ? hi : rx);
	uint32_t ry1 = ry + 1u;
	ry1 = ry1 < rx ? rx : (ry1 > hi ? hi : ry1);
	uint32_t num_bits = ry1 - rx;
	uint32_t range_mask = num_bits == 32u ? 0xffffffffu : ((1u << num_bits) - 1u) << (rx - start_index);
	return mask & range_mask;
}

static void deferred_lighting(const orc_gbuffer_t *g, const orc_camera_t *cam, const orc_cluster_params_t *p,
                              const orc_light_t *lights, const uint32_t *type_mask,
                              const uint32_t *bitmask, const uint32_t *cluster_range,
                              uint32_t *hdr_out, int32_t *out_tile_index, int32_t *out_z_index,
                              int32_t *out_light_count, int y0, int y1, const orc_shadows_t *shadows, int hdr_fp16)
{
	/* hdr_fp16 ("renderTargetFp16", scene_viewer_application.cpp:880-884): emissive / HDR-main are R16G16B16A16_SFLOAT;
	 * each of the two additive blends then rounds to fp16 (RNE), alpha passes through (the shaders write RGB only). */
	const uint16_t *emissive16 = (const uint16_t *)(const void *)g->emissive;
	uint16_t *hdr_out16 = (uint16_t *)(void *)hdr_out;
	const int W = g->width, H = g->height;
	const float *ivp = cam->inv_view_projection;
	const vec3 camera_pos = v3(cam->camera_position[0], cam->camera_position[1], cam->camera_position[2]);
	const vec3 dir_color = v3(g->dir_color[0], g->dir_color[1], g->dir_color[2]);
	const vec3 dir_dir = v3(g->dir_direction[0], g->dir_direction[1], g->dir_direction[2]);
	/* push.inv_resolution = 1 / viewport (renderer.cpp:1101-1102, 1120) */
	const float inv_res_x = 1.0f / (float)W, inv_res_y = 1.0f / (float)H;

#pragma omp parallel for schedule(dynamic, 4)
	for (int y = y0; y < y1; y++)
	{
		for (int x = 0; x < W; x++)
		{
			size_t idx = (size_t)y * W + x;
			float depth = g->depth[idx];
			uint32_t dst = hdr_fp16 ? 0u : g->emissive[idx];
			vec3 dst16 = v3(0.0f, 0.0f, 0.0f);
			if (hdr_fp16)
			{
				dst16 = v3(f16_to_f32(emissive16[4 * idx]), f16_to_f32(emissive16[4 * idx + 1]), f16_to_f32(emissive16[4 * idx + 2]));
				hdr_out16[4 * idx + 3] = emissive16[4 * idx + 3];
			}
			if (out_tile_index) out_tile_index[idx] = -1;
			if (out_z_index) out_z_index[idx] = -1;
			if (out_light_count) out_light_count[idx] = 0;
			if (depth == 0.0f)
			{
				/* depth test NOT_EQUAL fails: sky keeps the attachment value */
				if (hdr_fp16)
					for (int c = 0; c < 3; c++)
						hdr_out16[4 * idx + c] = emissive16[4 * idx + c];
				else
					hdr_out[idx] = dst;
				continue;
			}

			/* G-buffer decode (clustering.frag:32-35) */
			uint32_t a8 = g->albedo[idx];
			vec3 base_color = v3(srgb8_to_linear(a8 & 0xffu), srgb8_to_linear((a8 >> 8) & 0xffu), srgb8_to_linear((a8 >> 16) & 0xffu));
			float ambient_a = (float)(a8 >> 24) / 255.0f;
			uint32_t n10 = g->normal[idx];
			vec3 N = v3((float)(n10 & 0x3ffu) / 1023.0f * 2.0f - 1.0f,
			            (float)((n10 >> 10) & 0x3ffu) / 1023.0f * 2.0f - 1.0f,
			            (float)((n10 >> 20) & 0x3ffu) / 1023.0f * 2.0f - 1.0f);
			uint16_t mr = g->pbr[idx];
			float metallic = (float)(mr & 0xffu) / 255.0f;
			float roughness = (float)(mr >> 8) / 255.0f;

			/* clustering.vert:10-14 + quad: vClip = invVP * (ndc.xy, 0, 1), interpolated at the
			 * pixel centre; ndc = 2 * (frag + 0.5) / size - 1.  Evaluated per pixel as
			 * ((col0*ndc.x + col1*ndc.y) + col3)  (col2 * 0 dropped). */
			float ndc_x = 2.0f * ((float)x + 0.5f) * inv_res_x - 1.0f;
			float ndc_y = 2.0f * ((float)y + 0.5f) * inv_res_y - 1.0f;
			vec4 vclip = v4(ivp[0] * ndc_x + ivp[4] * ndc_y + ivp[12],
			                ivp[1] * ndc_x + ivp[5] * ndc_y + ivp[13],
			                ivp[2] * ndc_x + ivp[6] * ndc_y + ivp[14],
			                ivp[3] * ndc_x + ivp[7] * ndc_y + ivp[15]);
			/* clustering.frag:38-39 */
			vec4 clip = v4(vclip.x + depth * ivp[8], vclip.y + depth * ivp[9], vclip.z + depth * ivp[10], vclip.w + depth * ivp[11]);
			vec3 pos = v3(clip.x / clip.w, clip.y / clip.w, clip.z / clip.w);

			/* ---- draw 1: directional.frag:40-65 (LIGHTING_NO_AMBIENT, no SHADOWS,
			 * VOLUMETRIC_DIFFUSE_FALLBACK, no AMBIENT_OCCLUSION => base_ambient = 1) ---- */
			vec3 V = v3_normalize(v3_sub(camera_pos, pos));
			vec3 lit = brdf_terms(base_color, N, metallic, roughness, dir_dir, V, &dir_color);
			const float base_ambient = 1.0f;
			(void)ambient_a; /* material_ambient_factor only feeds the !LIGHTING_NO_AMBIENT branch */
			lit = v3_add(lit, v3(base_ambient * base_color.x * 0.05f, base_ambient * base_color.y * 0.05f, base_ambient * base_color.z * 0.05f));
			vec3 d = hdr_fp16 ? dst16 : unpack_r11g11b10(dst);
			if (hdr_fp16)
			{
				vec3 sum = v3_add(lit, d);
				dst16 = v3(f16_to_f32(f32_to_f16_rne(sum.x)), f16_to_f32(f32_to_f16_rne(sum.y)), f16_to_f32(f32_to_f16_rne(sum.z)));
			}
			else
				dst = pack_r11g11b10(v3_add(lit, d));

			/* ---- draw 2: clustering.frag + clusterer_bindless.h:29-84 ---- */
			vec3 result = v3(0.0f, 0.0f, 0.0f);
			/* gl_FragCoord.xy * inv_resolution * cluster.xy_scale */
			int cx = (int)(((float)x + 0.5f) * inv_res_x * p->xy_scale[0]);
			int cy = (int)(((float)y + 0.5f) * inv_res_y * p->xy_scale[1]);
			cx = cx < 0 ? 0 : (cx > p->resolution_xy[0] - 1 ? p->resolution_xy[0] - 1 : cx);
			cy = cy < 0 ? 0 : (cy > p->resolution_xy[1] - 1 ? p->resolution_xy[1] - 1 : cy);
			int cluster_index = cy * p->resolution_xy[0] + cx;
			int cluster_base = cluster_index * p->num_lights_32;

			vec3 cbase = v3(p->camera_base[0], p->camera_base[1], p->camera_base[2]);
			vec3 cfront = v3(p->camera_front[0], p->camera_front[1], p->camera_front[2]);
			float z = v3_dot(v3_sub(pos, cbase), cfront);
			float zs = z * p->z_scale;
			/* int(float): truncation; saturate like the hardware F2I so huge/NaN values stay defined */
			int z_index = zs >= 2147483520.0f ? 2147483647 : (zs <= -2147483648.0f ? (-2147483647 - 1) : (zs != zs ? 0 : (int)zs));
			z_index = z_index < 0 ? 0 : (z_index > p->z_max_index ? p->z_max_index : z_index);
			uint32_t rx = cluster_range[2 * z_index], ry = cluster_range[2 * z_index + 1];
			if (out_tile_index) out_tile_index[idx] = cluster_index;
			if (out_z_index) out_z_index[idx] = z_index;

			/* The reference widens [z_start, z_end] and ORs masks across the subgroup purely for
			 * scalarisation; a light outside this pixel's own mask lies outside its radius and
			 * contributes exactly +0, so the per-pixel form below is the same function. */
			int z_start = (int)(rx >> 5u);
			int z_end = (int)(ry >> 5u);
			int count = 0;
			for (int i = z_start; i <= z_end && i < p->num_lights_32; i++)
			{
				uint32_t mask = bitmask[cluster_base + i];
				mask = cluster_mask_range(mask, rx, ry, 32u * (uint32_t)i);
				uint32_t tm = type_mask[i];
				while (mask != 0u)
				{
					int bit = __builtin_ctz(mask);
					int index = 32 * i + bit;
					light_shadow_t sh = { 0, 0, 0, 0 };
					if (shadows && shadows->maps[index])
					{
						sh.transform = shadows->transforms + 16 * (size_t)index;
						sh.map = shadows->maps[index];
						sh.res = shadows->resolution;
						sh.wide = shadows->pcf_wide;
					}
					vec3 c = compute_positional_light(&lights[index], (tm >> bit) & 1u, base_color, N, metallic, roughness, pos, camera_pos, sh);
					result = v3_add(result, c);
					count++;
					mask &= ~(1u << bit);
				}
			}
			if (out_light_count) out_light_count[idx] = count;
			if (hdr_fp16)
			{
				vec3 sum = v3_add(result, dst16);
				hdr_out16[4 * idx] = f32_to_f16_rne(sum.x);
				hdr_out16[4 * idx + 1] = f32_to_f16_rne(sum.y);
				hdr_out16[4 * idx + 2] = f32_to_f16_rne(sum.z);
			}
			else
			{
				d = unpack_r11g11b10(dst);
				hdr_out[idx] = pack_r11g11b10(v3_add(result, d));
			}
		}
	}
}

void orc_deferred_lighting(const orc_gbuffer_t *g, const orc_camera_t *cam, const orc_cluster_params_t *p,
                           const orc_light_t *lights, const uint32_t *type_mask,
                           const uint32_t *bitmask, const uint32_t *cluster_range,
                           uint32_t *hdr_out, int32_t *out_tile_index, int32_t *out_z_index,
                           int32_t *out_light_count, int y0, int y1)
{
	deferred_lighting(g, cam, p, lights, type_mask, bitmask, cluster_range, hdr_out, out_tile_index, out_z_index, out_light_count, y0, y1, 0, 0);
}

/* the same pass with POSITIONAL_LIGHTS_SHADOW (clustering.frag through point.h:45-74, spot.h:51-77) */
void orc_deferred_lighting_shadowed(const orc_gbuffer_t *g, const orc_camera_t *cam, const orc_cluster_params_t *p,
                                    const orc_light_t *lights, const uint32_t *type_mask,
                                    const uint32_t *bitmask, const uint32_t *cluster_range, const orc_shadows_t *shadows,
                                    uint32_t *hdr_out, int y0, int y1)
{
	deferred_lighting(g, cam, p, lights, type_mask, bitmask, cluster_range, hdr_out, 0, 0, 0, y0, y1, shadows, 0);
}

/* "renderTargetFp16": g->emissive points at R16G16B16A16_SFLOAT texels (4 x uint16 per pixel), hdr_out likewise;
 * shadows may be NULL */
void orc_deferred_lighting_fp16(const orc_gbuffer_t *g, const orc_camera_t *cam, const orc_cluster_params_t *p,
                                const orc_light_t *lights, const uint32_t *type_mask,
                                const uint32_t *bitmask, const uint32_t *cluster_range, const orc_shadows_t *shadows,
                                uint16_t *hdr_out_rgba16f, int y0, int y1)
{
	deferred_lighting(g, cam, p, lights, type_mask, bitmask, cluster_range, (uint32_t *)(void *)hdr_out_rgba16f, 0, 0, 0, y0, y1, shadows, 1);
}

/* renderer.cpp:1009-1011: additive blend, the attachment store quantises (oracle_math.h pack_r11g11b10) */
void orc_blend_add_r11g11b10(uint32_t *dst, const float *src_rgb, const uint8_t *mask, int64_t count)
{
	for (int64_t i = 0; i < count; i++)
	{
		if (!mask[i])
			continue;
		vec3 d = unpack_r11g11b10(dst[i]);
		dst[i] = pack_r11g11b10(v3(d.x + src_rgb[3 * i + 0], d.y + src_rgb[3 * i + 1], d.z + src_rgb[3 * i + 2]));
	}
}

/* the same blend into an R16G16B16A16_SFLOAT attachment: RGB = fp16_rne(decode(dst) + src), alpha untouched */
void orc_blend_add_rgba16f(uint16_t *dst, const float *src_rgb, const uint8_t *mask, int64_t count)
{
	for (int64_t i = 0; i < count; i++)
	{
		if (!mask[i])
			continue;
		for (int c = 0; c < 3; c++)
			dst[4 * i + c] = f32_to_f16_rne(f16_to_f32(dst[4 * i + c]) + src_rgb[3 * i + c]);
	}
}

/* ---------------------------------------------------------------------------------------------
 * Volumetric fog, first pass: fog_light_density.comp (VolumetricFog::build_light_density, renderer/lights/
 * volumetric_fog.cpp:142-228) in its base variant -- no fog regions (density 0.1), no temporal reprojection (the first
 * frame), no floor lighting, unshadowed directional light, clustered positional lights without shadows.  Per froxel:
 * dithered position -> world position, fog albedo, in-scattered light (directional + compute_cluster_scatter_light,
 * clusterer_bindless.h:158-203) -> RGBA16F.  mat4 * vec4 pairwise, as the generated reference code evaluates it.
 * --------------------------------------------------------------------------------------------- */
static vec4 m4_mul_v4_pairwise(const float *m, vec4 v)
{
	return v4((m[0] * v.x + m[4] * v.y) + (m[8] * v.z + m[12] * v.w), (m[1] * v.x + m[5] * v.y) + (m[9] * v.z + m[13] * v.w),
	          (m[2] * v.x + m[6] * v.y) + (m[10] * v.z + m[14] * v.w), (m[3] * v.x + m[7] * v.y) + (m[11] * v.z + m[15] * v.w));
}

/* clusterer_bindless.h:158-203 with point.h:83-89 / spot.h:86-92 (a subgroup of one: the pixel's own mask) */
static vec3 cluster_scatter_light(const orc_cluster_params_t *p, const orc_light_t *lights, const uint32_t *type_mask, const uint32_t *bitmask,
                                  const uint32_t *cluster_range, vec3 world_pos, vec3 camera_pos)
{
	vec3 result = v3(0.0f, 0.0f, 0.0f);
	vec4 clip = m4_mul_v4_pairwise(p->transform, v4(world_pos.x, world_pos.y, world_pos.z, 1.0f));
	if (clip.w <= 0.0f)
		return result;
	float cxf = (clip.x * p->xy_scale[0]) / clip.w, cyf = (clip.y * p->xy_scale[1]) / clip.w;
	int cx = cxf >= 2147483520.0f ? 2147483647 : (cxf <= -2147483648.0f ? (-2147483647 - 1) : (cxf != cxf ? 0 : (int)cxf));
	int cy = cyf >= 2147483520.0f ? 2147483647 : (cyf <= -2147483648.0f ? (-2147483647 - 1) : (cyf != cyf ? 0 : (int)cyf));
	cx = cx < 0 ? 0 : (cx > p->resolution_xy[0] - 1 ? p->resolution_xy[0] - 1 : cx);
	cy = cy < 0 ? 0 : (cy > p->resolution_xy[1] - 1 ? p->resolution_xy[1] - 1 : cy);
	const int cluster_base = (cy * p->resolution_xy[0] + cx) * p->num_lights_32;
	vec3 cbase = v3(p->camera_base[0], p->camera_base[1], p->camera_base[2]), cfront = v3(p->camera_front[0], p->camera_front[1], p->camera_front[2]);
	float zs = v3_dot(v3_sub(world_pos, cbase), cfront) * p->z_scale;
	int z_index = zs >= 2147483520.0f ? 2147483647 : (zs <= -2147483648.0f ? (-2147483647 - 1) : (zs != zs ? 0 : (int)zs));
	z_index = z_index < 0 ? 0 : (z_index > p->z_max_index ? p->z_max_index : z_index);
	uint32_t rx = cluster_range[2 * z_index], ry = cluster_range[2 * z_index + 1];
	for (int i = (int)(rx >> 5u); i <= (int)(ry >> 5u) && i < p->num_lights_32; i++)
	{
		uint32_t mask = cluster_mask_range(bitmask[cluster_base + i], rx, ry, 32u * (uint32_t)i);
		const uint32_t tm = type_mask[i];
		while (mask != 0u)
		{
			const int bit = __builtin_ctz(mask);
			const orc_light_t *l = &lights[32 * i + bit];
			const light_shadow_t none = { 0, 0, 0, 0 };
			vec3 light_dir;
			vec3 color = ((tm >> bit) & 1u) ? compute_point_color(l, world_pos, &light_dir, none) : compute_spot_color(l, world_pos, &light_dir, none);
			float VoL = v3_dot(v3_normalize(v3_sub(camera_pos, world_pos)), v3_normalize(v3_sub(v3(l->position[0], l->position[1], l->position[2]), world_pos)));
			float phase = 0.55f - 0.45f * VoL;
			result = v3_add(result, v3(color.x * phase, color.y * phase, color.z * phase));
			mask &= ~(1u << bit);
		}
	}
	return result;
}

void orc_fog_light_density(const orc_fog_params_t *f, const orc_camera_t *cam, const orc_cluster_params_t *p, const orc_light_t *lights,
                           const uint32_t *type_mask, const uint32_t *bitmask, const uint32_t *cluster_range, const float *dir_color3,
                           const float *dir_direction3, const float *slice_extents, const uint32_t *dither_lut_rgba8, uint16_t *out_rgba16f)
{
	const int W = f->width, H = f->height, D = f->depth;
	const float inv_x = 1.0f / (float)W, inv_y = 1.0f / (float)H, inv_z = 1.0f / (float)D; /* volumetric_fog.cpp:165 */
	const vec3 camera_pos = v3(cam->camera_position[0], cam->camera_position[1], cam->camera_position[2]);
	const vec3 dir = v3(dir_direction3[0], dir_direction3[1], dir_direction3[2]);
	/* z_transform = (projection[2].zw, projection[3].zw); xy_scale = (inv_projection[0].x, inv_projection[1].y) (:161-168) */
	const float zt[4] = { cam->projection[10], cam->projection[11], cam->projection[14], cam->projection[15] };
	const float xy_scale[2] = { cam->inv_projection[0], cam->inv_projection[5] };
#pragma omp parallel for schedule(dynamic, 2)
	for (int z = 0; z < D; z++)
		for (int y = 0; y < H; y++)
			for (int x = 0; x < W; x++)
			{
				float u = ((float)x + 0.5f) * inv_x, v = ((float)y + 0.5f) * inv_y, w = ((float)z + 0.5f) * inv_z;
				const uint32_t dl = dither_lut_rgba8[((size_t)f->dither_offset * 128 + (size_t)(y & 127)) * 128 + (size_t)(x & 127)];
				float dx = (float)(dl & 255u) / 255.0f, dy = (float)((dl >> 8) & 255u) / 255.0f, dz = (float)((dl >> 16) & 255u) / 255.0f;
				dx -= 0.5f;
				dy -= 0.5f;
				dz = -dz;
				u += dx * inv_x;
				v += dy * inv_y;
				w += dz * inv_z;
				u = f_clamp(u, 0.0f, 1.0f);
				v = f_clamp(v, 0.0f, 1.0f);
				w = f_clamp(w, 0.001f, 1.0f);
				/* get_world_position */
				const float world_z = exp2f(w / f->slice_z_log2_scale) - 1.0f;
				const float zw_x = zt[2] - zt[0] * world_z, zw_y = zt[3] - zt[1] * world_z;
				const float clip_z = zw_x / zw_y;
				const vec4 clip = m4_mul_v4_pairwise(cam->inv_view_projection, v4(u * 2.0f - 1.0f, v * 2.0f - 1.0f, clip_z, 1.0f));
				const vec3 pos = v3(clip.x / clip.w, clip.y / clip.w, clip.z / clip.w);
				/* get_fog_albedo * compute_fog_density (no regions: 0.1) */
				const float lx = (u * 2.0f - 1.0f) * xy_scale[0], ly = (v * 2.0f - 1.0f) * xy_scale[1];
				const float length_mod = sqrtf(1.0f * 1.0f + lx * lx + ly * ly);
				/* texelFetch(uSliceExtents, int(gl_GlobalInvocationID.z)): the workgroup is 64 x 1 x 1 threads remapped to a 4 x 4 x 4
				 * box (.comp:207-215), so gl_GlobalInvocationID.z is the WORKGROUP's z index = z / 4, not the froxel's slice:
				 * four consecutive slices share the extent of slice z / 4.  Reproduced as the reference behaves. */
				float albedo = f->density_mod * slice_extents[z >> 2] * length_mod;
				albedo = albedo * 0.1f;
				/* compute_scatter_lighting (lighting_scatter.h:13-38) */
				const float VoL = v3_dot(v3_normalize(v3_sub(camera_pos, pos)), dir);
				const float phase = (0.55f - 0.45f * VoL) * 1.0f;
				vec3 s = v3(dir_color3[0] * phase, dir_color3[1] * phase, dir_color3[2] * phase);
				s = v3_add(s, cluster_scatter_light(p, lights, type_mask, bitmask, cluster_range, pos, camera_pos));
				uint16_t *o = out_rgba16f + 4 * (((size_t)z * H + y) * W + x);
				o[0] = f32_to_f16_rne(f->in_scatter_strength * s.x);
				o[1] = f32_to_f16_rne(f->in_scatter_strength * s.y);
				o[2] = f32_to_f16_rne(f->in_scatter_strength * s.z);
				o[3] = f32_to_f16_rne(albedo);
			}
}

/* VolumetricFog::compute_slice_extents (volumetric_fog.cpp:115-126) */
void orc_fog_slice_extents(int depth, float slice_z_log2_scale, float *out)
{
	for (int z = 0; z < depth; z++)
	{
		float end_z = exp2f(((float)z + 1.0f) / ((float)depth * slice_z_log2_scale)) - 1.0f;
		float start_z = exp2f((float)z / ((float)depth * slice_z_log2_scale)) - 1.0f;
		out[z] = end_z - start_z;
	}
}
