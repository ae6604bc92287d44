/*
 * oracle_post.c -- TEST INFRASTRUCTURE ONLY.  HDR post chain (K7..K11), FXAA (K12) and TAA
 * resolve (K13) restated from the reference GLSL under assets/shaders/post/.
 * See oracle_math.h for arithmetic rules.
 *
 * Sampling rules adopted (SURVEY.md §7 "Texture-unit semantics", §8c):
 *   - textureLod through LinearClamp on a DIFFERENT-size image: general bilinear with the
 *     normalised coordinate the shader computed ((x+0.5)*inv_out [+ off*inv_in]), see
 *     sample16f_linear();
 *   - textureLod at vUV on a SAME-size image at the pixel's own centre (tonemap's uHDR,
 *     FXAA/TAA centre and integer-offset taps, the FEEDBACK history tap): an exact texel
 *     fetch with clamp-to-edge (what a texture unit returns at a texel centre);
 *   - fragment-stage vUV := (x + 0.5) * (1 / W), (y + 0.5) * (1 / H) (quad.vert:10 interpolated).
 */
#include "oracle.h"
#include "oracle_math.h"

/* ---- K7: bloom_threshold.comp:23-45 ---- */
/* Storage format of the HDR image K7 / K11 / K13 read: 0 = B10G11R11_UFLOAT (default), 1 = R16G16B16A16_SFLOAT
 * ("renderTargetFp16").  Set by the *_fp16 entry points around the shared implementation (test infrastructure: one call
 * at a time). */
static int g_hdr_fp16 = 0;

static vec3 fetch_hdr(const uint32_t *hdr, int w, int h, int x, int y)
{
	x = x < 0 ? 0 : (x > w - 1 ? w - 1 : x);
	y = y < 0 ? 0 : (y > h - 1 ? h - 1 : y);
	if (g_hdr_fp16)
	{
		const uint16_t *t = (const uint16_t *)(const void *)hdr + 4 * ((size_t)y * w + x);
		return v3(f16_to_f32(t[0]), f16_to_f32(t[1]), f16_to_f32(t[2]));
	}
	return unpack_r11g11b10(hdr[(size_t)y * w + x]);
}

static vec3 sample_hdr_linear(const uint32_t *hdr, int w, int h, float u, float v)
{
	bilin_t s = bilin_setup(u, v, w, h);
	vec3 t00 = fetch_hdr(hdr, w, h, s.x0, s.y0), t10 = fetch_hdr(hdr, w, h, s.x1, s.y0);
	vec3 t01 = fetch_hdr(hdr, w, h, s.x0, s.y1), t11 = fetch_hdr(hdr, w, h, s.x1, s.y1);
	return v3(bilin_mix(t00.x, t10.x, t01.x, t11.x, s.a, s.b),
	          bilin_mix(t00.y, t10.y, t01.y, t11.y, s.a, s.b),
	          bilin_mix(t00.z, t10.z, t01.z, t11.z, s.a, s.b));
}

void orc_bloom_threshold(const uint32_t *hdr, int w_in, int h_in, const float *lum3,
                         uint16_t *out, int w, int h)
{
	/* hdr.cpp:138-141 */
	const float inv_x = 1.0f / (float)w, inv_y = 1.0f / (float)h;
#pragma omp parallel for
	for (int y = 0; y < h; y++)
	{
		for (int x = 0; x < w; x++)
		{
			float u = ((float)x + 0.5f) * inv_x, v = ((float)y + 0.5f) * inv_y;
			vec3 color = sample_hdr_linear(hdr, w_in, h_in, u, v);
			float luminance = f_max(f_max(color.x, color.y), color.z) + 0.0001f;
			float loglum = log2f(luminance);
			color = v3(color.x / luminance, color.y / luminance, color.z / luminance);
			if (lum3)
				luminance -= 8.0f * lum3[1];
			else
				luminance -= 8.0f;
			vec3 t = v3(f_max(color.x * luminance, 0.0f), f_max(color.y * luminance, 0.0f), f_max(color.z * luminance, 0.0f));
			store16f(out, w, x, y, v4(t.x, t.y, t.z, loglum));
		}
	}
}

/* 9-tap tent shared by K8 (off = 1.75) and K9 (off = 0.875): same tap order and weights as
 * bloom_downsample.comp:28-36 / bloom_upsample.comp:22-30. */
static vec4 tent9(img16f src, float u, float v, float off, float inv_in_x, float inv_in_y)
{
	static const float wgt[9] = { 0.25f, 0.0625f, 0.125f, 0.0625f, 0.125f, 0.125f, 0.0625f, 0.125f, 0.0625f };
	static const float ox[9] = { 0.0f, -1.0f, 0.0f, +1.0f, -1.0f, +1.0f, -1.0f, 0.0f, +1.0f };
	static const float oy[9] = { 0.0f, +1.0f, +1.0f, +1.0f, 0.0f, 0.0f, -1.0f, -1.0f, -1.0f };
	vec4 value = v4(0, 0, 0, 0);
	for (int k = 0; k < 9; k++)
	{
		/* vUV + vec2(ox*off, oy*off) * inv_input_size  (tap 0: vUV itself) */
		float tu = k == 0 ? u : u + (ox[k] * off) * inv_in_x;
		float tv = k == 0 ? v : v + (oy[k] * off) * inv_in_y;
		vec4 s = sample16f_linear(src, tu, tv);
		if (k == 0)
			value = v4(wgt[0] * s.x, wgt[0] * s.y, wgt[0] * s.z, wgt[0] * s.w);
		else
		{
			value.x += wgt[k] * s.x; value.y += wgt[k] * s.y; value.z += wgt[k] * s.z; value.w += wgt[k] * s.w;
		}
	}
	return value;
}

/* ---- K8: bloom_downsample.comp:21-42 ---- */
void orc_bloom_downsample(const uint16_t *in, int w_in, int h_in, const uint16_t *history, float lerp,
                          uint16_t *out, int w, int h)
{
	img16f src = { in, w_in, h_in };
	img16f hist = { history, w, h };
	const float inv_x = 1.0f / (float)w, inv_y = 1.0f / (float)h;            /* hdr.cpp:178-179 */
	const float inv_in_x = 1.0f / (float)w_in, inv_in_y = 1.0f / (float)h_in; /* hdr.cpp:180-181 */
#pragma omp parallel for
	for (int y = 0; y < h; y++)
	{
		for (int x = 0; x < w; x++)
		{
			float u = ((float)x + 0.5f) * inv_x, v = ((float)y + 0.5f) * inv_y;
			vec4 value = tent9(src, u, v, 1.75f, inv_in_x, inv_in_y);
			if (history)
			{
				/* mix(textureLod(uSamplerHistory, vUV), value, vec4(vec3(lerp), 1.0)); history is NearestClamp, same size */
				vec4 hs = fetch16f(hist, x, y);
				value = v4(f_mix(hs.x, value.x, lerp), f_mix(hs.y, value.y, lerp), f_mix(hs.z, value.z, lerp), f_mix(hs.w, value.w, 1.0f));
			}
			store16f(out, w, x, y, value);
		}
	}
}

/* ---- K9: bloom_upsample.comp:15-33 ---- */
void orc_bloom_upsample(const uint16_t *in, int w_in, int h_in, uint16_t *out, int w, int h)
{
	img16f src = { in, w_in, h_in };
	const float inv_x = 1.0f / (float)w, inv_y = 1.0f / (float)h;
	const float inv_in_x = 1.0f / (float)w_in, inv_in_y = 1.0f / (float)h_in;
#pragma omp parallel for
	for (int y = 0; y < h; y++)
	{
		for (int x = 0; x < w; x++)
		{
			float u = ((float)x + 0.5f) * inv_x, v = ((float)y + 0.5f) * inv_y;
			store16f(out, w, x, y, tent9(src, u, v, 0.875f, inv_in_x, inv_in_y));
		}
	}
}

/* ---- K10: luminance.comp:23-68, launched hdr.cpp:68-98 with size = d3 / 2 ---- */
void orc_luminance(const uint16_t *d3, int w, int h, float lerp, float min_loglum, float max_loglum,
                   float *lum3, float *grid)
{
	img16f src = { d3, w, h };
	int size_x = w / 2, size_y = h / 2;
	int iter_y = (size_y + 7) >> 3, iter_x = (size_x + 7) >> 3;
	float inv_size_x = 1.0f / (float)size_x, inv_size_y = 1.0f / (float)size_y;
	float shared_loglum[64];
	for (int ly = 0; ly < 8; ly++)
	{
		for (int lx = 0; lx < 8; lx++)
		{
			float total = 0.0f;
			for (int y = 0; y < iter_y; y++)
			{
				for (int x = 0; x < iter_x; x++)
				{
					int sx = x * 8 + lx, sy = y * 8 + ly;
					if (sx < size_x && sy < size_y)
					{
						float a = sample16f_linear(src, ((float)sx + 0.5f) * inv_size_x, ((float)sy + 0.5f) * inv_size_y).w;
						if (grid)
							grid[sy * size_x + sx] = a;
						total += a;
					}
				}
			}
			shared_loglum[ly * 8 + lx] = total; /* gl_LocalInvocationIndex = y*8 + x */
		}
	}
	for (int step = 32; step >= 2; step >>= 1)
		for (int i = 0; i < step; i++)
			shared_loglum[i] += shared_loglum[i + step];
	float loglum = shared_loglum[0] + shared_loglum[1];
	loglum *= inv_size_x * inv_size_y;
	loglum = f_clamp(loglum, min_loglum, max_loglum);
	float new_log_luma = f_mix(lum3[0], loglum, lerp);
	lum3[0] = new_log_luma;
	lum3[1] = exp2f(new_log_luma);
	lum3[2] = exp2f(-new_log_luma);
}

/* ---- K11: tonemap.frag ---- */
static float uncharted2(float x)
{
	const float A = 0.15f, B = 0.50f, C = 0.10f, D = 0.20f, E = 0.02f, F = 0.30f;
	/* The shader compiler (glslang) folds the constant sub-expressions C*B, D*E, D*F, E/F in DOUBLE
	 * precision from the decimal literals and then rounds once to fp32 -- e.g. D*F = 0.06 ->
	 * 0x3d75c28f, not 0.2f*0.3f = 0x3d75c290 (pinned by tests/test_oracle_ref_post_shaders.py). */
	const float CB = (float)(0.10 * 0.50), DE = (float)(0.20 * 0.02), DF = (float)(0.20 * 0.30), EF = (float)(0.02 / 0.30);
	(void)C; (void)D; (void)E; (void)F;
	return ((x * (A * x + CB) + DE) / (x * (A * x + B) + DF)) - EF;
}

void orc_tonemap(const uint32_t *hdr, int w, int h, const uint16_t *bloom, int bw, int bh,
                 const float *lum3, float exposure, int target_srgb, uint32_t *out, int y0, int y1)
{
	img16f bl = { bloom, bw, bh };
	const float inv_x = 1.0f / (float)w, inv_y = 1.0f / (float)h;
	const float white_scale = 1.0f / uncharted2(11.2f);
	const float k = lum3 ? (lum3[2] * exposure) : exposure;
#pragma omp parallel for
	for (int y = y0; y < y1; y++)
	{
		for (int x = 0; x < w; x++)
		{
			vec3 color = fetch_hdr(hdr, w, h, x, y);
			float u = ((float)x + 0.5f) * inv_x, v = ((float)y + 0.5f) * inv_y;
			vec4 b = sample16f_linear(bl, u, v);
			color = v3(color.x + b.x, color.y + b.y, color.z + b.z);
			color = v3(color.x * k, color.y * k, color.z * k);
			vec3 t = v3(uncharted2(color.x) * white_scale, uncharted2(color.y) * white_scale, uncharted2(color.z) * white_scale);
			/* colour attachment is R8G8B8A8_SRGB (application_headless.cpp:207) or, before a UNORM-reading AA pass,
			 * R8G8B8A8_UNORM; vec3 output => alpha 1 */
			if (target_srgb)
				out[(size_t)y * w + x] = linear_to_srgb8(t.x) | (linear_to_srgb8(t.y) << 8) | (linear_to_srgb8(t.z) << 16) | 0xff000000u;
			else
				out[(size_t)y * w + x] = float_to_unorm8(t.x) | (float_to_unorm8(t.y) << 8) | (float_to_unorm8(t.z) << 16) | 0xff000000u;
		}
	}
}

/* ---- K12: fxaa.frag:20-67; input is the sRGB image viewed as UNORM (fxaa.cpp:43) ---- */
static vec3 fetch_unorm8(const uint32_t *im, int w, int h, int x, int y)
{
	x = x < 0 ? 0 : (x > w - 1 ? w - 1 : x);
	y = y < 0 ? 0 : (y > h - 1 ? h - 1 : y);
	uint32_t p = im[(size_t)y * w + x];
	return v3((float)(p & 0xffu) / 255.0f, (float)((p >> 8) & 0xffu) / 255.0f, (float)((p >> 16) & 0xffu) / 255.0f);
}

static vec3 sample_unorm8_linear(const uint32_t *im, int w, int h, float u, float v)
{
	bilin_t s = bilin_setup(u, v, w, h);
	vec3 t00 = fetch_unorm8(im, w, h, s.x0, s.y0), t10 = fetch_unorm8(im, w, h, s.x1, s.y0);
	vec3 t01 = fetch_unorm8(im, w, h, s.x0, s.y1), t11 = fetch_unorm8(im, w, h, s.x1, s.y1);
	return v3(bilin_mix(t00.x, t10.x, t01.x, t11.x, s.a, s.b),
	          bilin_mix(t00.y, t10.y, t01.y, t11.y, s.a, s.b),
	          bilin_mix(t00.z, t10.z, t01.z, t11.z, s.a, s.b));
}

/* inc/srgb.h:4-10 */
static float decode_srgb1(float c)
{
	float small_side = c / 12.92f;
	float pow_side = powf((c + 0.055f) / 1.055f, 2.4f);
	float r = c <= 0.0404482362771082f ? small_side : pow_side;
	return f_clamp(r, 0.0f, 1.0f);
}

void orc_fxaa(const uint32_t *in, int w, int h, int target_srgb, uint32_t *out, int y0, int y1)
{
	const float FXAA_REDUCE_MIN = 1.0f / 128.0f, FXAA_REDUCE_MUL = 1.0f / 8.0f, FXAA_SPAN_MAX = 8.0f;
	const float inv_x = 1.0f / (float)w, inv_y = 1.0f / (float)h;
	const vec3 luma = v3(0.299f, 0.587f, 0.114f);
#pragma omp parallel for
	for (int y = y0; y < y1; y++)
	{
		for (int x = 0; x < w; x++)
		{
			float u = ((float)x + 0.5f) * inv_x, v = ((float)y + 0.5f) * inv_y;
			vec3 rgbNW = fetch_unorm8(in, w, h, x - 1, y - 1);
			vec3 rgbNE = fetch_unorm8(in, w, h, x + 1, y - 1);
			vec3 rgbSW = fetch_unorm8(in, w, h, x - 1, y + 1);
			vec3 rgbSE = fetch_unorm8(in, w, h, x + 1, y + 1);
			vec3 texColor = fetch_unorm8(in, w, h, x, y);
			float lumaNW = v3_dot(rgbNW, luma), lumaNE = v3_dot(rgbNE, luma);
			float lumaSW = v3_dot(rgbSW, luma), lumaSE = v3_dot(rgbSE, luma);
			float lumaM = v3_dot(texColor, luma);
			float lumaMin = f_min(lumaM, f_min(f_min(lumaNW, lumaNE), f_min(lumaSW, lumaSE)));
			float lumaMax = f_max(lumaM, f_max(f_max(lumaNW, lumaNE), f_max(lumaSW, lumaSE)));
			float dx = -((lumaNW + lumaNE) - (lumaSW + lumaSE));
			float dy = ((lumaNW + lumaSW) - (lumaNE + lumaSE));
			float dirReduce = f_max((lumaNW + lumaNE + lumaSW + lumaSE) * (0.25f * FXAA_REDUCE_MUL), FXAA_REDUCE_MIN);
			float rcpDirMin = 1.0f / (f_min(fabsf(dx), fabsf(dy)) + dirReduce);
			dx = f_clamp(dx * rcpDirMin, -FXAA_SPAN_MAX, FXAA_SPAN_MAX) * inv_x;
			dy = f_clamp(dy * rcpDirMin, -FXAA_SPAN_MAX, FXAA_SPAN_MAX) * inv_y;
			/* folded by glslang in double precision, then rounded: +-0.16666667163372039794921875 */
			const float k0 = (float)(1.0 / 3.0 - 0.5), k1 = (float)(2.0 / 3.0 - 0.5);
			vec3 a0 = sample_unorm8_linear(in, w, h, u + dx * k0, v + dy * k0);
			vec3 a1 = sample_unorm8_linear(in, w, h, u + dx * k1, v + dy * k1);
			vec3 rgbA = v3(0.5f * (a0.x + a1.x), 0.5f * (a0.y + a1.y), 0.5f * (a0.z + a1.z));
			vec3 b0 = sample_unorm8_linear(in, w, h, u + dx * -0.5f, v + dy * -0.5f);
			vec3 b1 = sample_unorm8_linear(in, w, h, u + dx * 0.5f, v + dy * 0.5f);
			vec3 rgbB = v3(rgbA.x * 0.5f + 0.25f * (b0.x + b1.x), rgbA.y * 0.5f + 0.25f * (b0.y + b1.y), rgbA.z * 0.5f + 0.25f * (b0.z + b1.z));
			float lumaB = v3_dot(rgbB, luma);
			vec3 color = ((lumaB < lumaMin) || (lumaB > lumaMax)) ? rgbA : rgbB;
			uint32_t r, g, b;
			if (target_srgb)
			{
				/* decode_srgb() then the sRGB attachment re-encodes on store */
				r = linear_to_srgb8(decode_srgb1(color.x));
				g = linear_to_srgb8(decode_srgb1(color.y));
				b = linear_to_srgb8(decode_srgb1(color.z));
			}
			else
			{
				r = float_to_unorm8(color.x); g = float_to_unorm8(color.y); b = float_to_unorm8(color.z);
			}
			out[(size_t)y * w + x] = r | (g << 8) | (b << 16) | 0xff000000u;
		}
	}
}

/* ---- K13: taa_resolve.frag + reprojection.h + reprojection_color_space.h ---- */
static vec3 taa_tonemap(vec3 c)
{
	c = v3(c.x * 8.0f, c.y * 8.0f, c.z * 8.0f);
	float r = 1.0f / (f_max(c.x, f_max(c.y, c.z)) + 1.0f);
	return v3(c.x * r, c.y * r, c.z * r);
}

static vec3 taa_tonemap_invert(vec3 c)
{
	float r = 1.0f / (1.0f - f_max(c.x, f_max(c.y, c.z)));
	/* (1/8) * c * RCP(...) left to right */
	return v3((1.0f / 8.0f) * c.x * r, (1.0f / 8.0f) * c.y * r, (1.0f / 8.0f) * c.z * r);
}

static vec3 rgb_to_ycgco(vec3 c)
{
	return v3(0.25f * c.x + 0.5f * c.y + 0.25f * c.z,
	          0.5f * c.y - 0.25f * c.x - 0.25f * c.z,
	          0.5f * c.x - 0.5f * c.z);
}

static vec3 ycgco_to_rgb(vec3 c)
{
	float tmp = c.x - c.y;
	return v3(tmp + c.z, c.x + c.y, tmp - c.z);
}

static vec3 hdr_to_taa(vec3 c) { return rgb_to_ycgco(taa_tonemap(c)); }

static vec3 taa_to_hdr(vec3 c)
{
	vec3 rgb = ycgco_to_rgb(c);
	rgb = v3(f_clamp(rgb.x, 0.0f, 0.999f), f_clamp(rgb.y, 0.0f, 0.999f), f_clamp(rgb.z, 0.0f, 0.999f));
	return taa_tonemap_invert(rgb);
}

/* reprojection.h:31-51 */
static vec3 clamp_box(vec3 color, vec3 lo, vec3 hi, int aabb)
{
	if (!aabb)
		return v3(f_clamp(color.x, lo.x, hi.x), f_clamp(color.y, lo.y, hi.y), f_clamp(color.z, lo.z, hi.z));
	vec3 center = v3(0.5f * (lo.x + hi.x), 0.5f * (lo.y + hi.y), 0.5f * (lo.z + hi.z));
	vec3 radius = v3(f_max(0.5f * (hi.x - lo.x), 0.0001f), f_max(0.5f * (hi.y - lo.y), 0.0001f), f_max(0.5f * (hi.z - lo.z), 0.0001f));
	vec3 v = v3_sub(color, center);
	vec3 units = v3(v.x / radius.x, v.y / radius.y, v.z / radius.z);
	float max_unit = f_max(f_max(fabsf(units.x), fabsf(units.y)), fabsf(units.z));
	if (max_unit > 1.0f)
		return v3(center.x + v.x / max_unit, center.y + v.y / max_unit, center.z + v.z / max_unit);
	return color;
}

typedef struct { const uint16_t *mv; const float *depth; int w, h; } taa_in;

static float fetch_depth(const taa_in *t, int x, int y)
{
	x = x < 0 ? 0 : (x > t->w - 1 ? t->w - 1 : x);
	y = y < 0 ? 0 : (y > t->h - 1 ? t->h - 1 : y);
	return t->depth[(size_t)y * t->w + x];
}

static vec2 fetch_mv(const taa_in *t, int x, int y)
{
	x = x < 0 ? 0 : (x > t->w - 1 ? t->w - 1 : x);
	y = y < 0 ? 0 : (y > t->h - 1 ? t->h - 1 : y);
	const uint16_t *p = t->mv + ((size_t)y * t->w + x) * 2;
	return v2(f16_to_f32(p[0]), f16_to_f32(p[1]));
}

/* reprojection.h:218-283 sample_nearest_velocity.  textureGather at UV - 0.5*inv_res covers
 * texels (x-1..x, y-1..y): .x=(x-1,y) .y=(x,y) .z=(x,y-1) .w=(x-1,y-1). */
static vec3 sample_nearest_velocity(const taa_in *t, int x, int y, int method_3x3)
{
	vec2 mv;
	float d;
#define TRY(px, py) do { float dd = fetch_depth(t, (px), (py)); if (dd > d) { mv = fetch_mv(t, (px), (py)); d = dd; } } while (0)
	if (method_3x3)
	{
		mv = fetch_mv(t, x + 1, y + 1);
		d = fetch_depth(t, x + 1, y + 1);
		/* quad0 = gather(ShiftUV): x,y,z,w */
		TRY(x - 1, y); TRY(x, y); TRY(x, y - 1); TRY(x - 1, y - 1);
		/* quad1 = gatherOffset(1,0).yz : (x+1,y), (x+1,y-1) */
		TRY(x + 1, y); TRY(x + 1, y - 1);
		/* quad2 = gatherOffset(0,1).xy : (x-1,y+1), (x,y+1) */
		TRY(x - 1, y + 1); TRY(x, y + 1);
	}
	else
	{
		/* 5-tap cross: quad0.xyz = (x-1,y),(x,y),(x,y-1); quad1 = gatherOffset(1,1).xz = (x,y+1),(x+1,y) */
		mv = fetch_mv(t, x - 1, y);
		d = fetch_depth(t, x - 1, y);
		TRY(x, y); TRY(x, y - 1); TRY(x, y + 1); TRY(x + 1, y);
	}
#undef TRY
	return v3(mv.x, mv.y, d);
}

static vec3 sample16f_rgb(img16f im, float u, float v)
{
	vec4 s = sample16f_linear(im, u, v);
	return v3(s.x, s.y, s.z);
}

/* reprojection.h:286-334 */
static vec3 sample_catmull_rom(img16f tex, float u, float v, const float *rt)
{
	float spx = u * rt[2], spy = v * rt[3];
	float t1x = floorf(spx - 0.5f) + 0.5f, t1y = floorf(spy - 0.5f) + 0.5f;
	float fx = spx - t1x, fy = spy - t1y;
#define W0(f) ((f) * (-0.5f + (f) * (1.0f - 0.5f * (f))))
#define W1(f) (1.0f + (f) * (f) * (-2.5f + 1.5f * (f)))
#define W2(f) ((f) * (0.5f + (f) * (2.0f - 1.5f * (f))))
#define W3(f) ((f) * (f) * (-0.5f + 0.5f * (f)))
	float w0x = W0(fx), w1x = W1(fx), w2x = W2(fx), w3x = W3(fx);
	float w0y = W0(fy), w1y = W1(fy), w2y = W2(fy), w3y = W3(fy);
#undef W0
#undef W1
#undef W2
#undef W3
	float w12x = w1x + w2x, w12y = w1y + w2y;
	float o12x = w2x / (w1x + w2x), o12y = w2y / (w1y + w2y);
	float t0x = (t1x - 1.0f) * rt[0], t0y = (t1y - 1.0f) * rt[1];
	float t3x = (t1x + 2.0f) * rt[0], t3y = (t1y + 2.0f) * rt[1];
	float t12x = (t1x + o12x) * rt[0], t12y = (t1y + o12y) * rt[1];
	vec3 result = v3(0, 0, 0);
#define ACC(uu, vv, wa, wb) do { vec4 s4 = sample16f_linear_snap(tex, (uu), (vv)); vec3 s = v3(s4.x, s4.y, s4.z); \
		result.x += s.x * (wa) * (wb); result.y += s.y * (wa) * (wb); result.z += s.z * (wa) * (wb); } while (0)
	ACC(t0x, t0y, w0x, w0y);
	ACC(t12x, t0y, w12x, w0y);
	ACC(t3x, t0y, w3x, w0y);
	ACC(t0x, t12y, w0x, w12y);
	ACC(t12x, t12y, w12x, w12y);
	ACC(t3x, t12y, w3x, w12y);
	ACC(t0x, t3y, w0x, w3y);
	ACC(t12x, t3y, w12x, w3y);
	ACC(t3x, t3y, w3x, w3y);
#undef ACC
	return result;
}

void orc_taa_resolve(const uint32_t *hdr, const float *depth, const uint16_t *mv, const uint16_t *history,
                     int w, int h, const float *reproj, int quality,
                     uint32_t *out_color, uint16_t *out_history, int y0, int y1)
{
	/* taa_resolve.frag:5-22 */
	const int cubic = quality == 2;
	const int clamp_aabb = quality != 0;
	const int nearest_3x3 = quality == 2;
	const float rt[4] = { 1.0f / (float)w, 1.0f / (float)h, (float)w, (float)h }; /* temporal.cpp:245-248 */
	taa_in tin = { mv, depth, w, h };
	img16f hist = { history, w, h };
#pragma omp parallel for
	for (int y = y0; y < y1; y++)
	{
		for (int x = 0; x < w; x++)
		{
			size_t idx = (size_t)y * w + x;
#define CUR(dx, dy) hdr_to_taa(fetch_hdr(hdr, w, h, x + (dx), y + (dy)))
			vec3 current = CUR(0, 0);
			vec3 out_c;
			if (!history)
			{
				out_c = current;
			}
			else
			{
				float u = ((float)x + 0.5f) * rt[0], v = ((float)y + 0.5f) * rt[1];
				vec3 MV_d = sample_nearest_velocity(&tin, x, y, nearest_3x3);
				float old_u, old_v;
				if (MV_d.x == 0.0f && MV_d.y == 0.0f)
				{
					vec4 clip = v4(2.0f * u - 1.0f, 2.0f * v - 1.0f, MV_d.z, 1.0f);
					vec4 rp = m4_mul_v4(reproj, clip);
					old_u = rp.x / rp.w;
					old_v = rp.y / rp.w;
					MV_d.x = u - old_u;
					MV_d.y = v - old_v;
				}
				else
				{
					old_u = u - MV_d.x;
					old_v = v - MV_d.y;
				}
				vec3 history_color = cubic ? sample_catmull_rom(hist, old_u, old_v, rt) : sample16f_rgb(hist, old_u, old_v);
				float MV_length = v2_length(v2(MV_d.x, MV_d.y));
				float MV_fast = f_min(MV_length * 50.0f, 1.0f);
				float gamma = f_mix(1.5f, 0.5f, MV_fast);
				history_color = v3(f_clamp(history_color.x, 0.0f, 1.0f), f_clamp(history_color.y, -1.0f, 1.0f), f_clamp(history_color.z, -1.0f, 1.0f));
				float lerp_factor = (1.0f + 2.0f * MV_fast) / 16.0f;

				/* clamp_history_box, reprojection.h:107-183 */
				vec3 c11 = current;
				vec3 c01 = CUR(-1, 0), c21 = CUR(+1, 0), c10 = CUR(0, -1), c12 = CUR(0, +1);
				vec3 lo = c11, hi = c11;
				if (quality == 0 || quality == 1)
				{
					lo = v3_min(lo, c01); lo = v3_min(lo, c21); lo = v3_min(lo, c10); lo = v3_min(lo, c12);
					hi = v3_max(hi, c01); hi = v3_max(hi, c21); hi = v3_max(hi, c10); hi = v3_max(hi, c12);
				}
				if (quality >= 1)
				{
					vec3 corner_lo = lo, corner_hi = hi;
					vec3 c00 = CUR(-1, -1), c22 = CUR(+1, +1), c02 = CUR(-1, +1), c20 = CUR(+1, -1);
					if (quality == 1)
					{
						lo = v3_min(lo, c00); lo = v3_min(lo, c22); lo = v3_min(lo, c02); lo = v3_min(lo, c20);
						hi = v3_max(hi, c00); hi = v3_max(hi, c22); hi = v3_max(hi, c02); hi = v3_max(hi, c20);
						lo = v3(0.5f * (corner_lo.x + lo.x), 0.5f * (corner_lo.y + lo.y), 0.5f * (corner_lo.z + lo.z));
						hi = v3(0.5f * (corner_hi.x + hi.x), 0.5f * (corner_hi.y + hi.y), 0.5f * (corner_hi.z + hi.z));
					}
					else
					{
						/* NEED_VARIANCE, reprojection.h:162-180 */
#define M1(c) ((c00.c + 2.0f * c01.c + c02.c + 2.0f * c10.c + 4.0f * c11.c + 2.0f * c12.c + c20.c + 2.0f * c21.c + c22.c) / 16.0f)
#define M2(c) (c00.c * c00.c + 2.0f * c01.c * c01.c + c02.c * c02.c + 2.0f * c10.c * c10.c + 4.0f * c11.c * c11.c + 2.0f * c12.c * c12.c + c20.c * c20.c + 2.0f * c21.c * c21.c + c22.c * c22.c)
						vec3 m1 = v3(M1(x), M1(y), M1(z));
						vec3 m2 = v3(M2(x), M2(y), M2(z));
#undef M1
#undef M2
						vec3 sigma = v3(sqrtf(f_max(m2.x / 16.0f - m1.x * m1.x, 0.0f)),
						                sqrtf(f_max(m2.y / 16.0f - m1.y * m1.y, 0.0f)),
						                sqrtf(f_max(m2.z / 16.0f - m1.z * m1.z, 0.0f)));
						lo = v3(m1.x - gamma * sigma.x, m1.y - gamma * sigma.y, m1.z - gamma * sigma.z);
						hi = v3(m1.x + gamma * sigma.x, m1.y + gamma * sigma.y, m1.z + gamma * sigma.z);
					}
				}
				history_color = clamp_box(history_color, lo, hi, clamp_aabb);
				out_c = v3_mixf(history_color, current, lerp_factor);
			}
#undef CUR
			vec3 color = taa_to_hdr(out_c);
			out_color[idx] = pack_r11g11b10(color);
			/* HistoryColor is a vec3 output on an RGBA16F attachment: alpha takes the default 1.0 */
			store16f(out_history, w, x, y, v4(out_c.x, out_c.y, out_c.z, 1.0f));
		}
	}
}

/* ---- K14: pq10_encode.frag ---- */
static float pq_channel(float nits)
{
	/* encode_pq (pq10_encode.frag:20-32); the constants are exact binary fractions */
	const float c1 = 0.8359375f, c2 = 18.8515625f, c3 = 18.6875f, m1 = 0.1593017578125f, m2 = 78.84375f;
	float y = nits / 10000.0f;
	float p = powf(y, m1);
	float num = c1 + c2 * p;
	float den = 1.0f + c3 * p;
	return powf(num / den, m2);
}

static uint32_t unorm10(float c)
{
	if (!(c > 0.0f)) c = 0.0f; /* also NaN (pow of a negative colour after the primaries conversion) */
	if (c > 1.0f) c = 1.0f;
	return (uint32_t)floorf(c * 1023.0f + 0.5f);
}

void orc_pq10_encode(const uint32_t *hdr, const uint32_t *ui, int w, int h, const float *m, float hdr_pre_exposure,
                     float ui_pre_exposure, float max_light_level, uint32_t *out, int y0, int y1)
{
	const float inv_max = 1.0f / max_light_level; /* hdr.cpp:637 */
	(void)h;
#pragma omp parallel for
	for (int y = y0; y < y1; y++)
		for (int x = 0; x < w; x++)
		{
			size_t i = (size_t)y * w + x;
			vec3 c = unpack_r11g11b10(hdr[i]);
			uint32_t u = ui[i];
			float ur = (float)(u & 0xffu) / 255.0f, ug = (float)((u >> 8) & 0xffu) / 255.0f, ub = (float)((u >> 16) & 0xffu) / 255.0f, ua = (float)(u >> 24) / 255.0f;
			float s = hdr_pre_exposure * ua;
			vec3 col = v3(c.x * s + ur * ui_pre_exposure, c.y * s + ug * ui_pre_exposure, c.z * s + ub * ui_pre_exposure);
			/* mat3(primary_conversion) * col: columns summed left to right */
			col = v3(m[0] * col.x + m[4] * col.y + m[8] * col.z, m[1] * col.x + m[5] * col.y + m[9] * col.z, m[2] * col.x + m[6] * col.y + m[10] * col.z);
			col = v3(col.x * inv_max, col.y * inv_max, col.z * inv_max);
			float k[3] = { col.x, col.y, col.z };
			for (int j = 0; j < 3; j++)
			{
				float ck = k[j] * 4.0f;
				float saturated = ck / (1.0f + ck);
				k[j] = k[j] > 0.75f ? saturated : k[j]; /* mix(col, saturated, greaterThan(col, 0.75)) */
				k[j] = pq_channel(k[j] * max_light_level);
			}
			out[i] = unorm10(k[0]) | (unorm10(k[1]) << 10) | (unorm10(k[2]) << 20) | (3u << 30);
		}
}

/* ---- "renderTargetFp16": the same three passes over an RGBA16F HDR image ---- */
void orc_bloom_threshold_fp16(const uint16_t *hdr_rgba16f, int w_in, int h_in, const float *lum3, uint16_t *out, int w, int h)
{
	g_hdr_fp16 = 1;
	orc_bloom_threshold((const uint32_t *)(const void *)hdr_rgba16f, w_in, h_in, lum3, out, w, h);
	g_hdr_fp16 = 0;
}

void orc_tonemap_fp16(const uint16_t *hdr_rgba16f, int w, int h, const uint16_t *bloom, int bw, int bh, const float *lum3, float exposure,
                      int target_srgb, uint32_t *out, int y0, int y1)
{
	g_hdr_fp16 = 1;
	orc_tonemap((const uint32_t *)(const void *)hdr_rgba16f, w, h, bloom, bw, bh, lum3, exposure, target_srgb, out, y0, y1);
	g_hdr_fp16 = 0;
}

void orc_taa_resolve_fp16(const uint16_t *hdr_rgba16f, const float *depth, const uint16_t *mv, const uint16_t *history, int w, int h,
                          const float *reproj16, int quality, uint32_t *out_color, uint16_t *out_history, int y0, int y1)
{
	g_hdr_fp16 = 1;
	orc_taa_resolve((const uint32_t *)(const void *)hdr_rgba16f, depth, mv, history, w, h, reproj16, quality, out_color, out_history, y0, y1);
	g_hdr_fp16 = 0;
}
