// grb_post_fast.cu -- the full-resolution streaming passes of the post chain (tonemap, FXAA, TAA
// resolve) arranged for instruction issue: at 3840x2160 each of them moves 66 - 265 MB (20 - 80 us
// at the H100 SXM's 3.35 TB/s data-sheet bandwidth) but the straightforward one-thread-per-pixel
// forms in grb_post.cu execute 130 - 1750 instructions per pixel.
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

// =============================================================================== K13 TAA resolve
// taa_resolve.frag:43-83 + reprojection.h at TAA_QUALITY 2 with history (the steady-state variant;
// the other variants stay on grb_post.cu's kernel).  A CTA owns 32x16 pixels.  Every texel of the tile
// plus a 1-pixel border is converted ONCE to float4(Y, Cg, Co, depth) in shared memory -- the 3x3
// neighbourhood statistics and the nearest-depth search then cost nine 16-byte shared-memory reads
// per pixel instead of nine HDR decodes + tonemaps + colour-space conversions and nine depth loads.
// The Catmull-Rom history fetch (nine bilinear taps in the shader) is evaluated as a separable
// weighted sum over the texels those taps touch, with the taps' positions formed by the shader's own
// arithmetic (see the comment at the filter).
// Per-texel colour-space conversions keep the shader's association (their chroma passes through zero);
// the filters are fused multiply-adds.
namespace grb
{
namespace
{
constexpr int kTaaTileW = 32, kTaaTileH = 16;
constexpr int kTaaSmemW = kTaaTileW + 2, kTaaSmemH = kTaaTileH + 2;

struct TaaFastArgs
{
	View<const uint32_t> hdr;
	View<const float> depth;
	View<const uint32_t> mv;
	View<const uint2> history;
	View<uint32_t> out_color;
	View<uint2> out_history;
	float m[16];
	int y0, y1;
	float inv_w, inv_h, w, h;
};

// HDRColorSpaceToTAA (reprojection_color_space.h:15-53) in the shader's own association, IEEE
// division, no contraction: it runs once per tile texel, and the chroma it produces passes
// through zero, where a reassociated sum would be off by many ulps of the (tiny) result.
GRB_DEV float3 hdr_to_taa_fast(uint32_t packed)
{
	float3 c = unpack_r11g11b10(packed);
	c = make_float3(fmul(c.x, 8.0f), fmul(c.y, 8.0f), fmul(c.z, 8.0f));
	const float r = fdiv(1.0f, fadd(fmax_(c.x, fmax_(c.y, c.z)), 1.0f));
	c = make_float3(fmul(c.x, r), fmul(c.y, r), fmul(c.z, r));
	return make_float3(fadd(fadd(fmul(0.25f, c.x), fmul(0.5f, c.y)), fmul(0.25f, c.z)), fsub(fsub(fmul(0.5f, c.y), fmul(0.25f, c.x)), fmul(0.25f, c.z)),
	                   fsub(fmul(0.5f, c.x), fmul(0.5f, c.z)));
}

GRB_DEV float3 fetch_hist(const View<const uint2> &im, int x, int y)
{
	const uint2 t = __ldg(&im.at(iclamp(x, 0, im.w - 1), iclamp(y, 0, im.h - 1)));
	const f2 rg = __half22float2(*reinterpret_cast<const __half2 *>(&t.x));
	return make_float3(rg.x, rg.y, __half2float(__ushort_as_half((unsigned short)(t.y & 0xffffu))));
}

__global__ void __launch_bounds__(256) taa_fast_kernel(const TaaFastArgs a)
{
	__shared__ float4 tile[kTaaSmemW * kTaaSmemH]; // 9.8 KB
	const int ox0 = blockIdx.x * kTaaTileW, oy0 = a.y0 + blockIdx.y * kTaaTileH;
	for (int i = threadIdx.x; i < kTaaSmemW * kTaaSmemH; i += 256)
	{
		const int ly = i / kTaaSmemW, lx = i - ly * kTaaSmemW;
		const int gx = iclamp(ox0 + lx - 1, 0, a.hdr.w - 1), gy = iclamp(oy0 + ly - 1, 0, a.hdr.h - 1);
		const float3 c = hdr_to_taa_fast(__ldg(&a.hdr.at(gx, gy)));
		tile[i] = make_float4(c.x, c.y, c.z, __ldg(&a.depth.at(gx, gy)));
	}
	__syncthreads();
	const int lx = threadIdx.x & (kTaaTileW - 1);
	const int x = ox0 + lx;
	if (x >= a.out_color.w)
		return;
#pragma unroll 1
	for (int ly = threadIdx.x / kTaaTileW; ly < kTaaTileH; ly += 256 / kTaaTileW)
	{
		const int y = oy0 + ly;
		if (y >= a.y1)
			break;
		const float4 *c = tile + (ly + 1) * kTaaSmemW + (lx + 1);
		const float4 c00 = c[-kTaaSmemW - 1], c10 = c[-kTaaSmemW], c20 = c[-kTaaSmemW + 1];
		const float4 c01 = c[-1], c11 = c[0], c21 = c[1];
		const float4 c02 = c[kTaaSmemW - 1], c12 = c[kTaaSmemW], c22 = c[kTaaSmemW + 1];
		// sample_nearest_velocity (reprojection.h:218-283), 3x3: start at (+1,+1), then the gather order
		int sel = 8; // index = (dy + 1) * 3 + (dx + 1)
		float d = c22.w;
#define GRB_TRY(T, IDX) if ((T).w > d) { d = (T).w; sel = (IDX); }
		GRB_TRY(c01, 3) GRB_TRY(c11, 4) GRB_TRY(c10, 1) GRB_TRY(c00, 0) GRB_TRY(c21, 5) GRB_TRY(c20, 2) GRB_TRY(c02, 6) GRB_TRY(c12, 7)
#undef GRB_TRY
		const int sdy = sel / 3 - 1, sdx = sel - (sel / 3) * 3 - 1;
		const uint32_t mvp = __ldg(&a.mv.at(iclamp(x + sdx, 0, a.hdr.w - 1), iclamp(y + sdy, 0, a.hdr.h - 1)));
		float mvx = __half2float(__ushort_as_half((unsigned short)(mvp & 0xffffu))), mvy = __half2float(__ushort_as_half((unsigned short)(mvp >> 16)));
		const float u = ((float)x + 0.5f) * a.inv_w, v = ((float)y + 0.5f) * a.inv_h;
		float old_u, old_v;
		if (mvx == 0.0f && mvy == 0.0f)
		{
			// The history position is formed with the shader's association and IEEE division: an ulp of u is
			// 1e-4 texel at 4K, and the Catmull-Rom weights amplify it by the local contrast of the history.
			const float cx = fsub(fmul(2.0f, u), 1.0f), cy = fsub(fmul(2.0f, v), 1.0f);
			const float *m = a.m;
			const float px = fadd(fadd(fadd(fmul(m[0], cx), fmul(m[4], cy)), fmul(m[8], d)), m[12]);
			const float py = fadd(fadd(fadd(fmul(m[1], cx), fmul(m[5], cy)), fmul(m[9], d)), m[13]);
			const float pw = fadd(fadd(fadd(fmul(m[3], cx), fmul(m[7], cy)), fmul(m[11], d)), m[15]);
			old_u = fdiv(px, pw);
			old_v = fdiv(py, pw);
			mvx = fsub(u, old_u);
			mvy = fsub(v, old_v);
		}
		else
		{
			old_u = fsub(u, mvx);
			old_v = fsub(v, mvy);
		}
		// Catmull-Rom, reprojection.h:286-334.  The shader takes 9 bilinear samples at (t0, t12, t3) x
		// (t0, t12, t3): t0 and t3 aim at texel centres, t12 lies between two texels.  The positions are
		// formed with the shader's own operations (they pass through normalised coordinates); a tap within
		// 2^-9 texel of a centre IS that texel (snap_weight, grb_common.cuh -- a sampler's fixed-point position
		// has 8 fractional bits), so per axis the taps name four texels: one for t0, two for t12, one for
		// t3, and the 9 samples collapse to a separable 4 x 4 weighted sum.
		float3 hist;
		{
			const float spx = fmul(old_u, a.w), spy = fmul(old_v, a.h);
			const float t1x = fadd(floorf(fsub(spx, 0.5f)), 0.5f), t1y = fadd(floorf(fsub(spy, 0.5f)), 0.5f);
			const float fx = fsub(spx, t1x), fy = fsub(spy, t1y);
			int sx[4], sy[4];
			float wxs[4], wys[4];
			auto axis_slots = [](float t1, float f, float inv_n, float n_f, int n, int *slot, float *wgt) {
				// weights of the four Catmull-Rom taps (shader expressions, left to right, no contraction)
				const float w0 = fmul(f, fadd(-0.5f, fmul(f, fsub(1.0f, fmul(0.5f, f)))));
				const float w1 = fadd(1.0f, fmul(fmul(f, f), fadd(-2.5f, fmul(1.5f, f))));
				const float w2 = fmul(f, fadd(0.5f, fmul(f, fsub(2.0f, fmul(1.5f, f)))));
				const float w3 = fmul(fmul(f, f), fadd(-0.5f, fmul(0.5f, f)));
				const float w12 = fadd(w1, w2);
				const float o12 = fdiv(w2, w12);
				// LinearClamp along this axis (grb_common.cuh bilin_setup) for the three positions
				auto locate = [&](float pos, int &i, float &frac) {
					const float g = fsub(fmul(pos, n_f), 0.5f);
					float fl = floorf(g);
					frac = snap_weight(fsub(g, fl));
					fl = fclamp(fl, -2.0f, n_f + 1.0f);
					i = (int)fl;
				};
				int i0, i12, i3;
				float f0, f12, f3;
				locate(fmul(fsub(t1, 1.0f), inv_n), i0, f0);
				locate(fmul(fadd(t1, o12), inv_n), i12, f12);
				locate(fmul(fadd(t1, 2.0f), inv_n), i3, f3);
				// t0 / t3: snapped to one texel (for any image up to 8192 texels wide the position is within
				// 2^-10 of a centre; a weight that did not snap keeps its larger share -- never taken there)
				slot[0] = iclamp(f0 >= 0.5f ? i0 + 1 : i0, 0, n - 1);
				wgt[0] = w0;
				slot[1] = iclamp(i12, 0, n - 1);
				wgt[1] = w12 * (1.0f - f12);
				slot[2] = iclamp(i12 + 1, 0, n - 1);
				wgt[2] = w12 * f12;
				slot[3] = iclamp(f3 >= 0.5f ? i3 + 1 : i3, 0, n - 1);
				wgt[3] = w3;
			};
			axis_slots(t1x, fx, a.inv_w, a.w, a.history.w, sx, wxs);
			axis_slots(t1y, fy, a.inv_h, a.h, a.history.h, sy, wys);
			f2 acc_yg = mk2(0.0f);
			float acc_o = 0.0f;
#pragma unroll
			for (int j = 0; j < 4; j++)
			{
				const uint2 *rowp = a.history.p + (size_t)sy[j] * a.history.pitch;
				f2 row_yg = mk2(0.0f);
				float row_o = 0.0f;
#pragma unroll
				for (int i = 0; i < 4; i++)
				{
					const uint2 raw = __ldg(rowp + sx[i]);
					const f2 rg = __half22float2(*reinterpret_cast<const __half2 *>(&raw.x));
					const float o = __half2float(__ushort_as_half((unsigned short)(raw.y & 0xffffu)));
					row_yg = fma2(mk2(wxs[i]), rg, row_yg);
					row_o = fmaf(wxs[i], o, row_o);
				}
				acc_yg = fma2(mk2(wys[j]), row_yg, acc_yg);
				acc_o = fmaf(wys[j], row_o, acc_o);
			}
			hist = make_float3(acc_yg.x, acc_yg.y, acc_o);
		}
		const float mv_len = sqrtf(fmaf(mvx, mvx, mvy * mvy));
		const float mv_fast = fminf(mv_len * 50.0f, 1.0f);
		const float gamma = fmaf(0.5f, mv_fast, 1.5f * (1.0f - mv_fast));
		hist = make_float3(fminf(fmaxf(hist.x, 0.0f), 1.0f), fminf(fmaxf(hist.y, -1.0f), 1.0f), fminf(fmaxf(hist.z, -1.0f), 1.0f));
		const float lerp_factor = fmaf(2.0f, mv_fast, 1.0f) * (1.0f / 16.0f);

		// clamp_history_box, variance form (reprojection.h:107-183): weights 1 2 1 / 2 4 2 / 1 2 1.
		// m2 / 16 - m1^2 is a cancellation; in flat regions its value is rounding noise of either
		// evaluation order (sigma ~ 3e-4 of the mean), which bounds the clip box far inside one fp16 ulp.
		float3 m1, sigma;
		{
#define GRB_YG(T) make_float2((T).x, (T).y)
			const f2 corners = add2(add2(GRB_YG(c00), GRB_YG(c02)), add2(GRB_YG(c20), GRB_YG(c22)));
			const f2 edges = add2(add2(GRB_YG(c01), GRB_YG(c10)), add2(GRB_YG(c12), GRB_YG(c21)));
			const f2 s1 = fma2(mk2(4.0f), GRB_YG(c11), fma2(mk2(2.0f), edges, corners));
			f2 q_c = mul2(GRB_YG(c00), GRB_YG(c00));
			q_c = fma2(GRB_YG(c02), GRB_YG(c02), q_c); q_c = fma2(GRB_YG(c20), GRB_YG(c20), q_c); q_c = fma2(GRB_YG(c22), GRB_YG(c22), q_c);
			f2 q_e = mul2(GRB_YG(c01), GRB_YG(c01));
			q_e = fma2(GRB_YG(c10), GRB_YG(c10), q_e); q_e = fma2(GRB_YG(c12), GRB_YG(c12), q_e); q_e = fma2(GRB_YG(c21), GRB_YG(c21), q_e);
			const f2 s2 = fma2(mul2(mk2(4.0f), GRB_YG(c11)), GRB_YG(c11), fma2(mk2(2.0f), q_e, q_c));
#undef GRB_YG
			const float s1z = fmaf(4.0f, c11.z, fmaf(2.0f, (c01.z + c10.z) + (c12.z + c21.z), (c00.z + c02.z) + (c20.z + c22.z)));
			const float s2z = fmaf(4.0f * c11.z, c11.z, fmaf(2.0f, fmaf(c01.z, c01.z, fmaf(c10.z, c10.z, fmaf(c12.z, c12.z, c21.z * c21.z))),
			                                             fmaf(c00.z, c00.z, fmaf(c02.z, c02.z, fmaf(c20.z, c20.z, c22.z * c22.z)))));
			m1 = make_float3(s1.x * (1.0f / 16.0f), s1.y * (1.0f / 16.0f), s1z * (1.0f / 16.0f));
			sigma = make_float3(sqrtf(fmaxf(fmaf(s2.x, 1.0f / 16.0f, -m1.x * m1.x), 0.0f)), sqrtf(fmaxf(fmaf(s2.y, 1.0f / 16.0f, -m1.y * m1.y), 0.0f)),
			                    sqrtf(fmaxf(fmaf(s2z, 1.0f / 16.0f, -m1.z * m1.z), 0.0f)));
		}
		const float3 lo = make_float3(fmaf(-gamma, sigma.x, m1.x), fmaf(-gamma, sigma.y, m1.y), fmaf(-gamma, sigma.z, m1.z));
		const float3 hi = make_float3(fmaf(gamma, sigma.x, m1.x), fmaf(gamma, sigma.y, m1.y), fmaf(gamma, sigma.z, m1.z));
		// clamp_box (AABB clip towards the centre), reprojection.h:31-51
		{
			const float3 center = make_float3(0.5f * (lo.x + hi.x), 0.5f * (lo.y + hi.y), 0.5f * (lo.z + hi.z));
			const float3 radius = make_float3(fmaxf(0.5f * (hi.x - lo.x), 0.0001f), fmaxf(0.5f * (hi.y - lo.y), 0.0001f), fmaxf(0.5f * (hi.z - lo.z), 0.0001f));
			const float3 vv = make_float3(hist.x - center.x, hist.y - center.y, hist.z - center.z);
			const float max_unit = fmaxf(fmaxf(fabsf(vv.x) * rcp_fast(radius.x), fabsf(vv.y) * rcp_fast(radius.y)), fabsf(vv.z) * rcp_fast(radius.z));
			if (max_unit > 1.0f)
			{
				const float ru = rcp_fast(max_unit);
				hist = make_float3(fmaf(vv.x, ru, center.x), fmaf(vv.y, ru, center.y), fmaf(vv.z, ru, center.z));
			}
		}
		const float il = 1.0f - lerp_factor;
		const float3 out_c = make_float3(fmaf(c11.x, lerp_factor, hist.x * il), fmaf(c11.y, lerp_factor, hist.y * il), fmaf(c11.z, lerp_factor, hist.z * il));
		// TAAToHDRColorSpace (YCgCo -> RGB, clamp, inverse tonemap), shader association
		const float tmp = fsub(out_c.x, out_c.y);
		const float3 rgb = make_float3(fclamp(fadd(tmp, out_c.z), 0.0f, 0.999f), fclamp(fadd(out_c.x, out_c.y), 0.0f, 0.999f), fclamp(fsub(tmp, out_c.z), 0.0f, 0.999f));
		const float rr = fdiv(1.0f, fsub(1.0f, fmax_(rgb.x, fmax_(rgb.y, rgb.z))));
		a.out_color.at(x, y) = pack_r11g11b10(fmul(fmul(0.125f, rgb.x), rr), fmul(fmul(0.125f, rgb.y), rr), fmul(fmul(0.125f, rgb.z), rr));
		a.out_history.at(x, y) = pack_rgba16f(make_float4(out_c.x, out_c.y, out_c.z, 1.0f));
	}
}
} // namespace

bool launch_taa_fast(const GrbImage *hdr, const GrbImage *depth, const GrbImage *mv, const GrbImage *history, const float *reproj16, const GrbImage *out_color,
                     const GrbImage *out_history, GrbRows rows, cudaStream_t stream, int32_t *rc)
{
	// Opt-in (GRB_TAA_TILES=1): at 3840x2160 this kernel takes 556 us against 584 us for the exact kernel in
	// grb_post.cu -- 216 M instructions at 35 % issue utilisation, 16 warps per SM waiting on the history
	// loads behind the exact reprojection arithmetic -- which does not pay for giving up bit-exactness.
	// DESIGN.md section 8 says what would (a history tile in shared memory).
	const char *tiles = getenv("GRB_TAA_TILES");
	if (!tiles || tiles[0] == '0' || exact_requested() || hdr->width > 8192 || hdr->height > 8192)
		return false;
	TaaFastArgs a;
	a.hdr = view_of<const uint32_t>(hdr);
	a.depth = view_of<const float>(depth);
	a.mv = view_of<const uint32_t>(mv);
	a.history = view_of<const uint2>(history);
	a.out_color = view_of<uint32_t>(out_color);
	a.out_history = view_of<uint2>(out_history);
	for (int i = 0; i < 16; i++)
		a.m[i] = reproj16[i];
	a.y0 = rows.y0;
	a.y1 = rows.y1;
	a.inv_w = 1.0f / (float)hdr->width; // temporal.cpp:245-248
	a.inv_h = 1.0f / (float)hdr->height;
	a.w = (float)hdr->width;
	a.h = (float)hdr->height;
	dim3 grid((hdr->width + kTaaTileW - 1) / kTaaTileW, (rows.y1 - rows.y0 + kTaaTileH - 1) / kTaaTileH, 1);
	taa_fast_kernel<<<grid, 256, 0, stream>>>(a);
	*rc = check_launch("grb_taa_resolve");
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
