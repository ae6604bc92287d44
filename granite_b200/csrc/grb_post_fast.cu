// grb_post_fast.cu -- the full-resolution streaming passes of the post chain (tonemap, FXAA, HDR10
// PQ) arranged for instruction issue: at 3840x2160 each of them moves 66 - 100 MB (20 - 30 us
// at the H100 SXM's 3.35 TB/s data-sheet bandwidth) but the straightforward one-thread-per-pixel
// forms in grb_post.cu execute 130 or more instructions per pixel.
//
// Contract: every output is within 1 unit of its STORED format (8-bit code, B10G11R11 code, fp16
// ulp) of the reference arithmetic ("within 1 ULP per channel"), and identical for all but a
// ~1e-4 fraction of values: the arithmetic is re-associated and uses FMA and the fast
// reciprocal / log2 / exp2 units, none of which moves a result by more than a few fp32 ulps
// before it is quantised.  Two channels or pixels travel together in float2 lanes (f2 below).
// (Compiled with FMA contraction on; grb_post.cu keeps the bit-exact forms, selected with
// GRB_POST_EXACT=1 and used for shapes these kernels do not cover.)
#include "grb_common.cuh"

#include <cstdlib>

namespace grb
{
namespace
{
using f2 = float2;
GRB_DEV f2 mk2(float a) { return make_float2(a, a); }
// plain operators: ptxas may contract a multiply feeding an add into an FFMA, as the contract allows
GRB_DEV f2 add2(f2 a, f2 b) { return make_float2(a.x + b.x, a.y + b.y); }
GRB_DEV f2 sub2(f2 a, f2 b) { return make_float2(a.x - b.x, a.y - b.y); }
GRB_DEV f2 mul2(f2 a, f2 b) { return make_float2(a.x * b.x, a.y * b.y); }
GRB_DEV f2 fma2(f2 a, f2 b, f2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

// ------------------------------------------------------------------------------- K11 tonemap
// tonemap.frag:55-66.  One thread = 4 horizontally adjacent pixels of one row.  With the bloom image
// at exactly 1/4 resolution the four pixels share 3 columns x 2 rows of bloom texels and their
// bilinear weights are the constants 5/8, 7/8, 1/8, 3/8 (the sampler's own arithmetic lands within
// 2^-20 of them); rows likewise by y mod 4.
GRB_DEV f2 uncharted2_num(f2 x)
{
	const float A = 0.15f, CB = (float)(0.10 * 0.50), DE = (float)(0.20 * 0.02);
	return fma2(x, fma2(mk2(A), x, mk2(CB)), mk2(DE));
}
GRB_DEV f2 uncharted2_den(f2 x)
{
	const float A = 0.15f, B = 0.50f, DF = (float)(0.20 * 0.30);
	return fma2(x, fma2(mk2(A), x, mk2(B)), mk2(DF));
}

// 255 * OETF(saturate(c)) + 0.5, ready for truncation
GRB_DEV float srgb_scaled(float c)
{
	c = __saturatef(c);
	const float p = fmaf(ex2_fast(lg2_fast(c) * (1.0f / 2.4f)), 1.055f * 255.0f, -0.055f * 255.0f + 0.5f);
	return c <= 0.0031308f ? fmaf(c, 12.92f * 255.0f, 0.5f) : p;
}

template <bool DynamicExposure, bool SrgbTarget>
__global__ void __launch_bounds__(256) tonemap_fast_kernel(View<const uint32_t> hdr, View<const uint2> bloom, const float *__restrict__ lum, float exposure,
                                                           View<uint32_t> out, int y0, int y1)
{
	const int x4 = (blockIdx.x * 32 + threadIdx.x) * 4;
	const int y = y0 + blockIdx.y * 8 + threadIdx.y;
	if (x4 >= out.w || y >= y1)
		return;
	const uint4 h4 = __ldg(reinterpret_cast<const uint4 *>(&hdr.at(x4, y)));

	// bloom rows: centre (y + 0.5) / 4 - 0.5 -> floor = (y >> 2) - 1 for y mod 4 < 2, else y >> 2
	const int ym = y & 3;
	const int by = (y >> 2) - (ym < 2 ? 1 : 0);
	const float wb = ym == 0 ? 0.625f : (ym == 1 ? 0.875f : (ym == 2 ? 0.125f : 0.375f));
	const int r0 = iclamp(by, 0, bloom.h - 1), r1 = iclamp(by + 1, 0, bloom.h - 1);
	const int k = x4 >> 2;
	const int c0 = iclamp(k - 1, 0, bloom.w - 1), c2 = iclamp(k + 1, 0, bloom.w - 1);
	// vertical interpolation of the three columns (shared by the four pixels); (r, g) packed, b apart
	f2 col_rg[3];
	float col_b[3];
	{
		const int cols[3] = { c0, k, c2 };
#pragma unroll
		for (int i = 0; i < 3; i++)
		{
			const uint2 ta = __ldg(&bloom.at(cols[i], r0)), tb = __ldg(&bloom.at(cols[i], r1));
			const f2 a_rg = __half22float2(*reinterpret_cast<const __half2 *>(&ta.x)), b_rg = __half22float2(*reinterpret_cast<const __half2 *>(&tb.x));
			const float a_b = __half2float(__ushort_as_half((unsigned short)(ta.y & 0xffffu))), b_b = __half2float(__ushort_as_half((unsigned short)(tb.y & 0xffffu)));
			col_rg[i] = fma2(mk2(wb), sub2(b_rg, a_rg), a_rg);
			col_b[i] = fmaf(wb, b_b - a_b, a_b);
		}
	}
	const float kexp = DynamicExposure ? (__ldg(&lum[2]) * exposure) : exposure;
	const float EF = (float)(0.02 / 0.30);
	const float white_num = fmaf(11.2f, fmaf(0.15f, 11.2f, (float)(0.10 * 0.50)), (float)(0.20 * 0.02));
	const float white_den = fmaf(11.2f, fmaf(0.15f, 11.2f, 0.50f), (float)(0.20 * 0.30));
	const float white_scale = 1.0f / (white_num / white_den - EF);
	const uint32_t hp[4] = { h4.x, h4.y, h4.z, h4.w };
	uint32_t px[4];
#pragma unroll
	for (int j = 0; j < 4; j++)
	{
		const float wa = j == 0 ? 0.625f : (j == 1 ? 0.875f : (j == 2 ? 0.125f : 0.375f));
		const int i0 = j < 2 ? 0 : 1;
		const f2 b_rg = fma2(mk2(wa), sub2(col_rg[i0 + 1], col_rg[i0]), col_rg[i0]);
		const float b_b = fmaf(wa, col_b[i0 + 1] - col_b[i0], col_b[i0]);
		const float3 c = unpack_r11g11b10(hp[j]);
		const f2 x_rg = mul2(add2(make_float2(c.x, c.y), b_rg), mk2(kexp));
		const float x_b = (c.z + b_b) * kexp;
		// one reciprocal for the three channels: 1/d_i = (prod of the other two) / (d_r d_g d_b)
		const f2 n_rg = uncharted2_num(x_rg), d_rg = uncharted2_den(x_rg);
		const float n_b = fmaf(x_b, fmaf(0.15f, x_b, (float)(0.10 * 0.50)), (float)(0.20 * 0.02));
		const float d_b = fmaf(x_b, fmaf(0.15f, x_b, 0.50f), (float)(0.20 * 0.30));
		const float d_rg_prod = d_rg.x * d_rg.y;
		const float inv_all = rcp_fast(d_rg_prod * d_b);
		const float inv_rg_prod = inv_all * d_b;                              // 1 / (d_r d_g)
		const f2 q_rg = mul2(n_rg, mul2(make_float2(d_rg.y, d_rg.x), mk2(inv_rg_prod)));
		const float q_b = n_b * (inv_all * d_rg_prod);
		const f2 t_rg = fma2(q_rg, mk2(white_scale), mk2(-EF * white_scale));
		const float t_b = fmaf(q_b, white_scale, -EF * white_scale);
		if (SrgbTarget)
			px[j] = (uint32_t)__float2int_rz(srgb_scaled(t_rg.x)) | ((uint32_t)__float2int_rz(srgb_scaled(t_rg.y)) << 8) |
			        ((uint32_t)__float2int_rz(srgb_scaled(t_b)) << 16) | 0xff000000u;
		else
			px[j] = (uint32_t)__float2int_rz(fmaf(__saturatef(t_rg.x), 255.0f, 0.5f)) | ((uint32_t)__float2int_rz(fmaf(__saturatef(t_rg.y), 255.0f, 0.5f)) << 8) |
			        ((uint32_t)__float2int_rz(fmaf(__saturatef(t_b), 255.0f, 0.5f)) << 16) | 0xff000000u;
	}
	*reinterpret_cast<uint4 *>(&out.at(x4, y)) = make_uint4(px[0], px[1], px[2], px[3]);
}

bool exact_requested()
{
	static const bool on = getenv("GRB_POST_EXACT") != nullptr;
	return on;
}
} // namespace

// Launchers for the entry points in grb_post.cu; false = shape not covered (generic kernel runs).
bool launch_tonemap_fast(const GrbImage *hdr, const GrbImage *bloom, const float *luminance, float exposure, const GrbImage *out, GrbRows rows, cudaStream_t stream,
                         int32_t *rc)
{
	const bool ok = !exact_requested() && (out->width % 4) == 0 && bloom->width * 4 == out->width && bloom->height * 4 == out->height &&
	                (hdr->row_pitch % 16) == 0 && (out->row_pitch % 16) == 0 && (reinterpret_cast<uintptr_t>(hdr->data) % 16) == 0 &&
	                (reinterpret_cast<uintptr_t>(out->data) % 16) == 0;
	if (!ok)
		return false;
	const bool srgb = out->format == GRB_FORMAT_R8G8B8A8_SRGB;
	auto h = view_of<const uint32_t>(hdr);
	auto b = view_of<const uint2>(bloom);
	auto o = view_of<uint32_t>(out);
	dim3 block(32, 8), grid((out->width / 4 + 31) / 32, (rows.y1 - rows.y0 + 7) / 8, 1);
	if (luminance && srgb)
		tonemap_fast_kernel<true, true><<<grid, block, 0, stream>>>(h, b, luminance, exposure, o, rows.y0, rows.y1);
	else if (luminance)
		tonemap_fast_kernel<true, false><<<grid, block, 0, stream>>>(h, b, luminance, exposure, o, rows.y0, rows.y1);
	else if (srgb)
		tonemap_fast_kernel<false, true><<<grid, block, 0, stream>>>(h, b, nullptr, exposure, o, rows.y0, rows.y1);
	else
		tonemap_fast_kernel<false, false><<<grid, block, 0, stream>>>(h, b, nullptr, exposure, o, rows.y0, rows.y1);
	*rc = check_launch("grb_tonemap");
	return true;
}
} // namespace grb

// =============================================================================== K12 FXAA
// fxaa.frag:20-67.  A CTA owns 64x16 output pixels; the input tile plus a 5-pixel border (the four
// directional taps reach +-4 pixels, +1 for their bilinear footprint) is unpacked ONCE per texel into
// shared memory -- rgb as three fp16 (exact: 0..255 are integers) and the luma as fp32, in 0..255
// units -- with clamp-to-edge applied while filling, so nothing inside the tile clamps again.  (A
// float4 per texel made the 16 gathered texels per pixel a shared-memory bandwidth bound: 84
// wavefronts per warp; this layout needs 37.)  All of the shader's arithmetic is scale-invariant
// except the 1/128 floor of dirReduce, which is carried as 255/128.  An sRGB target applies
// decode_srgb and the attachment re-encodes on store: that pair is the identity on [0, 1] up to
// rounding, so both targets round the same value (difference from the reference: ties only, 1 code).
namespace grb
{
namespace
{
constexpr int kFxTileW = 64, kFxTileH = 16, kFxHalo = 5;
constexpr int kFxSmemW = kFxTileW + 2 * kFxHalo, kFxSmemH = kFxTileH + 2 * kFxHalo; // 74 x 26

GRB_DEV float byte_to_float(uint32_t word, int byte_index)
{
	// 0x4B000000 | byte is 2^23 + byte exactly
	const uint32_t bits = __byte_perm(word, 0x4B000000u, byte_index == 0 ? 0x7440 : (byte_index == 1 ? 0x7441 : 0x7442));
	return __uint_as_float(bits) - 8388608.0f;
}

struct Rgb
{
	f2 rg;
	float b;
};
GRB_DEV Rgb fx_load(const uint2 *p)
{
	const uint2 t = *p;
	Rgb c;
	c.rg = __half22float2(*reinterpret_cast<const __half2 *>(&t.x));
	c.b = __half2float(__ushort_as_half((unsigned short)(t.y & 0xffffu)));
	return c;
}

GRB_DEV Rgb fx_bilinear(const uint2 *tile, float fx, float fy)
{
	// (fx, fy): texel-space position relative to the tile origin (texel centres at integers)
	const float flx = floorf(fx), fly = floorf(fy);
	const float a = fx - flx, b = fy - fly;
	const uint2 *p = tile + (int)fly * kFxSmemW + (int)flx;
	const Rgb t00 = fx_load(p), t10 = fx_load(p + 1), t01 = fx_load(p + kFxSmemW), t11 = fx_load(p + kFxSmemW + 1);
	const f2 top_rg = fma2(mk2(a), sub2(t10.rg, t00.rg), t00.rg);
	const f2 bot_rg = fma2(mk2(a), sub2(t11.rg, t01.rg), t01.rg);
	const float top_b = fmaf(a, t10.b - t00.b, t00.b), bot_b = fmaf(a, t11.b - t01.b, t01.b);
	Rgb r;
	r.rg = fma2(mk2(b), sub2(bot_rg, top_rg), top_rg);
	r.b = fmaf(b, bot_b - top_b, top_b);
	return r;
}

__global__ void __launch_bounds__(256) fxaa_fast_kernel(View<const uint32_t> in, View<uint32_t> out, int y0, int y1)
{
	__shared__ uint2 tile[kFxSmemW * kFxSmemH];  // rgb as fp16 x 3 (+ pad): 15.4 KB
	__shared__ float luma[kFxSmemW * kFxSmemH];  // 7.7 KB
	const int ox0 = blockIdx.x * kFxTileW, oy0 = y0 + blockIdx.y * kFxTileH;
	for (int i = threadIdx.x; i < kFxSmemW * kFxSmemH; i += 256)
	{
		const int ly = i / kFxSmemW, lx = i - ly * kFxSmemW;
		const int gx = iclamp(ox0 + lx - kFxHalo, 0, in.w - 1), gy = iclamp(oy0 + ly - kFxHalo, 0, in.h - 1);
		const uint32_t p = __ldg(&in.at(gx, gy));
		const float r = byte_to_float(p, 0), g = byte_to_float(p, 1), b = byte_to_float(p, 2);
		const __half2 rg = __floats2half2_rn(r, g);
		uint2 t;
		t.x = *reinterpret_cast<const uint32_t *>(&rg);
		t.y = (uint32_t)__half_as_ushort(__float2half_rn(b));
		tile[i] = t;
		luma[i] = fmaf(b, 0.114f, fmaf(g, 0.587f, r * 0.299f));
	}
	__syncthreads();
	const int lx = threadIdx.x & (kFxTileW - 1);
	const int x = ox0 + lx;
	if (x >= out.w)
		return;
#pragma unroll 1
	for (int ly = threadIdx.x / kFxTileW; ly < kFxTileH; ly += 256 / kFxTileW)
	{
		const int y = oy0 + ly;
		if (y >= y1)
			break;
		const float *c = luma + (ly + kFxHalo) * kFxSmemW + (lx + kFxHalo);
		const float lumaNW = c[-kFxSmemW - 1], lumaNE = c[-kFxSmemW + 1], lumaSW = c[kFxSmemW - 1], lumaSE = c[kFxSmemW + 1], lumaM = c[0];
		const float lumaMin = fminf(lumaM, fminf(fminf(lumaNW, lumaNE), fminf(lumaSW, lumaSE)));
		const float lumaMax = fmaxf(lumaM, fmaxf(fmaxf(lumaNW, lumaNE), fmaxf(lumaSW, lumaSE)));
		float dx = -((lumaNW + lumaNE) - (lumaSW + lumaSE));
		float dy = (lumaNW + lumaSW) - (lumaNE + lumaSE);
		const float dirReduce = fmaxf((((lumaNW + lumaNE) + lumaSW) + lumaSE) * 0.03125f, 255.0f / 128.0f);
		const float rcpDirMin = rcp_fast(fminf(fabsf(dx), fabsf(dy)) + dirReduce);
		dx = fminf(fmaxf(dx * rcpDirMin, -8.0f), 8.0f); // in pixels
		dy = fminf(fmaxf(dy * rcpDirMin, -8.0f), 8.0f);
		const float bx = (float)(lx + kFxHalo), by = (float)(ly + kFxHalo);
		const float k0 = (float)(1.0 / 3.0 - 0.5), k1 = (float)(2.0 / 3.0 - 0.5);
		const Rgb a0 = fx_bilinear(tile, fmaf(dx, k0, bx), fmaf(dy, k0, by));
		const Rgb a1 = fx_bilinear(tile, fmaf(dx, k1, bx), fmaf(dy, k1, by));
		const Rgb b0 = fx_bilinear(tile, fmaf(dx, -0.5f, bx), fmaf(dy, -0.5f, by));
		const Rgb b1 = fx_bilinear(tile, fmaf(dx, 0.5f, bx), fmaf(dy, 0.5f, by));
		const f2 A_rg = mul2(mk2(0.5f), add2(a0.rg, a1.rg));
		const float A_b = 0.5f * (a0.b + a1.b);
		const f2 B_rg = fma2(mk2(0.25f), add2(b0.rg, b1.rg), mul2(A_rg, mk2(0.5f)));
		const float B_b = fmaf(0.25f, b0.b + b1.b, A_b * 0.5f);
		const float lumaB = fmaf(B_b, 0.114f, fmaf(B_rg.y, 0.587f, B_rg.x * 0.299f));
		const bool useA = (lumaB < lumaMin) || (lumaB > lumaMax);
		const float cr = useA ? A_rg.x : B_rg.x, cg = useA ? A_rg.y : B_rg.y, cb = useA ? A_b : B_b;
		const uint32_t r8 = (uint32_t)__float2int_rz(fminf(fmaxf(cr, 0.0f), 255.0f) + 0.5f);
		const uint32_t g8 = (uint32_t)__float2int_rz(fminf(fmaxf(cg, 0.0f), 255.0f) + 0.5f);
		const uint32_t b8 = (uint32_t)__float2int_rz(fminf(fmaxf(cb, 0.0f), 255.0f) + 0.5f);
		out.at(x, y) = r8 | (g8 << 8) | (b8 << 16) | 0xff000000u;
	}
}
} // namespace

bool launch_fxaa_fast(const GrbImage *in, const GrbImage *out, GrbRows rows, cudaStream_t stream, int32_t *rc)
{
	if (exact_requested())
		return false;
	dim3 grid((out->width + kFxTileW - 1) / kFxTileW, (rows.y1 - rows.y0 + kFxTileH - 1) / kFxTileH, 1);
	fxaa_fast_kernel<<<grid, 256, 0, stream>>>(view_of<const uint32_t>(in), view_of<uint32_t>(out), rows.y0, rows.y1);
	*rc = check_launch("grb_fxaa");
	return true;
}
} // namespace grb

// =============================================================================== K14 HDR10 / PQ
// pq10_encode.frag:20-52 (setup_hdr10_pq_encoding, renderer/post/hdr.cpp:595-658): scene colour +
// UI layer -> display primaries -> soft knee above 0.75 -> ST.2084 (PQ) -> A2B10G10R10.  Four pixels
// per thread, 16-byte loads and stores; the two pow() per channel are lg2 / ex2 (the output has 10 bits).
namespace grb
{
namespace
{
struct PqParams
{
	float m[9]; // column-major mat3
	float hdr_pre, ui_pre, max_light, inv_max;
};

GRB_DEV float pq_channel_fast(float col, float max_light)
{
	const float ck = col * 4.0f;
	const float knee = ck * rcp_fast(1.0f + ck);
	const float c = col > 0.75f ? knee : col;
	const float y = c * max_light * (1.0f / 10000.0f);
	// pow(y, m1): y <= 0 (black, or negative after the primaries conversion: NaN in the shader, stored as 0) -> 0
	const float p = y > 0.0f ? ex2_fast(lg2_fast(y) * 0.1593017578125f) : 0.0f;
	const float num = fmaf(18.8515625f, p, 0.8359375f), den = fmaf(18.6875f, p, 1.0f);
	const float n = ex2_fast(lg2_fast(num * rcp_fast(den)) * 78.84375f);
	return y >= 0.0f ? n : 0.0f;
}

__global__ void __launch_bounds__(256) pq10_encode_kernel(View<const uint32_t> hdr, View<const uint32_t> ui, PqParams q, View<uint32_t> out, int y0, int y1)
{
	const int x4 = (blockIdx.x * 32 + threadIdx.x) * 4;
	const int y = y0 + blockIdx.y * 8 + threadIdx.y;
	if (x4 >= out.w || y >= y1)
		return;
	uint32_t hp[4], up[4], px[4];
	if (x4 + 3 < out.w && (reinterpret_cast<uintptr_t>(&hdr.at(x4, y)) & 15u) == 0 && (reinterpret_cast<uintptr_t>(&ui.at(x4, y)) & 15u) == 0)
	{
		const uint4 h4 = __ldg(reinterpret_cast<const uint4 *>(&hdr.at(x4, y))), u4 = __ldg(reinterpret_cast<const uint4 *>(&ui.at(x4, y)));
		hp[0] = h4.x; hp[1] = h4.y; hp[2] = h4.z; hp[3] = h4.w;
		up[0] = u4.x; up[1] = u4.y; up[2] = u4.z; up[3] = u4.w;
	}
	else
		for (int j = 0; j < 4; j++)
		{
			const int xx = min(x4 + j, out.w - 1);
			hp[j] = __ldg(&hdr.at(xx, y));
			up[j] = __ldg(&ui.at(xx, y));
		}
#pragma unroll
	for (int j = 0; j < 4; j++)
	{
		const float3 c = unpack_r11g11b10(hp[j]);
		const float k255 = 1.0f / 255.0f;
		const float ur = (float)(up[j] & 0xffu) * k255, ug = (float)((up[j] >> 8) & 0xffu) * k255, ub = (float)((up[j] >> 16) & 0xffu) * k255,
		            ua = (float)(up[j] >> 24) * k255;
		const float s = q.hdr_pre * ua;
		const float r = fmaf(c.x, s, ur * q.ui_pre), g = fmaf(c.y, s, ug * q.ui_pre), b = fmaf(c.z, s, ub * q.ui_pre);
		const float cr = fmaf(q.m[6], b, fmaf(q.m[3], g, q.m[0] * r)) * q.inv_max;
		const float cg = fmaf(q.m[7], b, fmaf(q.m[4], g, q.m[1] * r)) * q.inv_max;
		const float cb = fmaf(q.m[8], b, fmaf(q.m[5], g, q.m[2] * r)) * q.inv_max;
		const uint32_t qr = (uint32_t)__float2int_rz(fmaf(__saturatef(pq_channel_fast(cr, q.max_light)), 1023.0f, 0.5f));
		const uint32_t qg = (uint32_t)__float2int_rz(fmaf(__saturatef(pq_channel_fast(cg, q.max_light)), 1023.0f, 0.5f));
		const uint32_t qb = (uint32_t)__float2int_rz(fmaf(__saturatef(pq_channel_fast(cb, q.max_light)), 1023.0f, 0.5f));
		px[j] = qr | (qg << 10) | (qb << 20) | (3u << 30);
	}
	if (x4 + 3 < out.w && (reinterpret_cast<uintptr_t>(&out.at(x4, y)) & 15u) == 0)
		*reinterpret_cast<uint4 *>(&out.at(x4, y)) = make_uint4(px[0], px[1], px[2], px[3]);
	else
		for (int j = 0; j < 4 && x4 + j < out.w; j++)
			out.at(x4 + j, y) = px[j];
}
} // namespace
} // namespace grb

using namespace grb;

extern "C" int32_t grb_pq10_encode(const GrbImage *hdr, const GrbImage *ui, const float *primary_conversion16, float hdr_pre_exposure, float ui_pre_exposure,
                                   float max_light_level, const GrbImage *out, GrbRows rows, void *stream)
{
	if (!image_ok(hdr, GRB_FORMAT_B10G11R11_UFLOAT_PACK32, 4) || !image_ok(ui, GRB_FORMAT_R8G8B8A8_UNORM, 4) ||
	    !image_ok(out, GRB_FORMAT_A2B10G10R10_UNORM_PACK32, 4) || !primary_conversion16 || !(max_light_level > 0.0f) || hdr->width != out->width ||
	    hdr->height != out->height || ui->width != out->width || ui->height != out->height)
	{
		set_last_error("grb_pq10_encode: hdr B10G11R11_UFLOAT, ui R8G8B8A8_UNORM, out A2B10G10R10_UNORM of one size; max_light_level > 0");
		return GRB_ERR_UNSUPPORTED_FORMAT;
	}
	rows = full_rows(rows, out->height);
	if (rows.y1 <= rows.y0)
		return GRB_OK;
	PqParams q;
	for (int c = 0; c < 3; c++)
		for (int r = 0; r < 3; r++)
			q.m[c * 3 + r] = primary_conversion16[c * 4 + r]; // mat3(mat4)
	q.hdr_pre = hdr_pre_exposure;
	q.ui_pre = ui_pre_exposure;
	q.max_light = max_light_level;
	q.inv_max = 1.0f / max_light_level; // hdr.cpp:637
	dim3 block(32, 8), grid((out->width + 127) / 128, (rows.y1 - rows.y0 + 7) / 8, 1);
	pq10_encode_kernel<<<grid, block, 0, as_stream(stream)>>>(view_of<const uint32_t>(hdr), view_of<const uint32_t>(ui), q, view_of<uint32_t>(out), rows.y0, rows.y1);
	return check_launch("grb_pq10_encode");
}
