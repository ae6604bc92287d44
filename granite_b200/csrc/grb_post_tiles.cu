// grb_post_tiles.cu -- the bloom pyramid as shared-memory tile kernels fed by TMA.
//
// The 9-tap tent filters of the bloom pyramid (bloom_downsample.comp:21-42, bloom_upsample.comp:15-33)
// read every source texel 2.25 .. 9 times.  The plain kernels in grb_post.cu leave that reuse to
// L1/L2 and pay for it in instructions: 36 dependent 8-byte loads, 36 index clamps and 9 bilinear
// set-ups per output texel.  Here a CTA owns a 32x16 tile of OUTPUT texels:
//
//   1. one elected thread issues a single `cp.async.bulk.tensor.2d` (TMA) for the rectangle of
//      source texels the tile can touch, completion on an mbarrier; out-of-image parts of the box
//      are zero-filled by the TMA unit and never read (indices are clamped to the image first, as
//      the sampler's clamp-to-edge demands);
//   2. the raw texels are widened once to fp32 in shared memory (each source texel is converted
//      once instead of once per tap);
//   3. every output texel then needs 3 column set-ups + 3 row set-ups (the taps' bilinear
//      footprints are separable) and 36 conflict-free 16-byte shared-memory reads; the arithmetic
//      is the sampler's fp32 sequence, two channels at a time in float2 lanes.  Each lane is an
//      explicitly rounded multiply or add (__fmul_rn / __fadd_rn), which ptxas never contracts, so
//      the sequence is the oracle's unfused one (the tests allow 1 fp16 ULP per channel).
//
// The first two passes of the chain are FUSED (grb_bloom_threshold_downsample): the 1/2-resolution
// threshold image "t" is produced tile by tile in shared memory from a TMA-loaded tile of HDR-main,
// rounded to fp16 exactly as the image store would round it, and consumed by the 1/4-resolution
// downsample in the same CTA.  The threshold arithmetic uses FMA, one reciprocal for the three
// colour / luminance quotients and the hardware log2: rgb and alpha within 1 fp16 ulp of the oracle.  t is only written to HBM when the caller asks for it, which removes
// its 16.6 MB write and 16.6 MB read per 4K frame.
//
// Eligibility (checked on the host, the generic kernels remain the fallback): exact 2:1 size
// steps, 16-byte aligned bases and pitches.  That covers every large level of the BASELINE
// configurations (4K: 3840 -> 1920 -> 960 -> 480 -> 240; only 240x135 -> 120x68 and back are not
// 2:1 and stay on the generic path, 0.3 MB).
#include "grb_common.cuh"
#include "grb_peer.cuh"

#include <cuda.h>

#include <cstdio>
#include <cstdlib>
#include <mutex>

namespace grb
{
namespace
{
using f2 = float2;
GRB_DEV f2 mk2(float a) { return make_float2(a, a); }
GRB_DEV f2 add2(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
GRB_DEV f2 mul2(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// ---------------------------------------------------------------------------------- TMA plumbing
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn()
{
	static EncodeTiledFn fn = nullptr;
	static std::once_flag once;
	std::call_once(once, [] {
		void *p = nullptr;
		cudaDriverEntryPointQueryResult q;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
			fn = reinterpret_cast<EncodeTiledFn>(p);
		else
			cudaGetLastError();
	});
	return fn;
}

// Tensor map over an image seen as rows of 32-bit words (an RGBA16F texel is two words).
bool make_map_u32(CUtensorMap *map, const GrbImage *im, int words_per_texel, int box_words, int box_rows)
{
	EncodeTiledFn fn = encode_fn();
	if (!fn)
		return false;
	if ((reinterpret_cast<uintptr_t>(im->data) & 15u) != 0 || (im->row_pitch & 15) != 0 || ((box_words * 4) & 15) != 0 || box_words > 256 || box_rows > 256)
		return false;
	cuuint64_t dims[2] = { (cuuint64_t)im->width * (cuuint64_t)words_per_texel, (cuuint64_t)im->height };
	cuuint64_t strides[1] = { (cuuint64_t)im->row_pitch };
	cuuint32_t box[2] = { (cuuint32_t)box_words, (cuuint32_t)box_rows };
	cuuint32_t estr[2] = { 1, 1 };
	return fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, im->data, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
	          CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

GRB_DEV uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

GRB_DEV void mbar_init(uint32_t bar)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// One elected thread: arm the barrier with the byte count of the box, start the copy.
GRB_DEV void tma_load_box(uint32_t dst, const CUtensorMap *map, int c0, int c1, uint32_t bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
	asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst), "l"(map),
	             "r"(c0), "r"(c1), "r"(bar)
	             : "memory");
}

GRB_DEV void mbar_wait(uint32_t bar, uint32_t parity)
{
	uint32_t done = 0;
	while (!done)
		asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2; selp.u32 %0, 1, 0, q; }" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
}

// ---------------------------------------------------------------------------------- tile geometry
constexpr int kThreads = 256;
constexpr int kOutW = 32, kOutH = 16; // output tile of every kernel here

// Down (source = 2 x output): taps at +-1.75 source texels around 2x + 0.5 touch texels 2x - 2 .. 2x + 3.
constexpr int kDownSrcW = 2 * kOutW + 4, kDownSrcH = 2 * kOutH + 4; // 68 x 36
// Up (output = 2 x source): taps at +-0.875 around x / 2 - 0.25 touch texels x/2 - 2 .. x/2 + 1 (+1 for odd x).
constexpr int kUpSrcW = kOutW / 2 + 4, kUpSrcH = kOutH / 2 + 4; // 20 x 12

// One axis of a LinearClamp sample at normalised coordinate c over n texels, local to a tile that
// starts at texel `origin` and holds `span` texels: the sampler's exact arithmetic (grb_common.cuh
// bilin_setup), indices clamped to the image and then made tile-relative.  The final min/max keeps a
// rounding surprise inside the tile's memory; it never binds when the geometry above is right.
struct Axis
{
	int i0, i1;
	float w;
};
// Down tiles store a row as [even columns | odd columns]: a warp's lanes read columns 2x + k, which
// would otherwise be a stride-2 (two-way bank conflict) pattern for 16-byte reads.
template <int SPAN, bool SPLIT>
GRB_DEV int col_slot(int c)
{
	return SPLIT ? ((c & 1) * (SPAN / 2) + (c >> 1)) : c;
}

GRB_DEV Axis axis_setup(float c, int n, int origin, int span)
{
	Axis a;
	float f = fsub(fmul(c, (float)n), 0.5f);
	float fl = floorf(f);
	a.w = fsub(f, fl);
	fl = fclamp(fl, -2.0f, (float)n + 1.0f);
	if (!(fl == fl)) fl = 0.0f;
	int i = (int)fl;
	a.i0 = iclamp(iclamp(i, 0, n - 1) - origin, 0, span - 1);
	a.i1 = iclamp(iclamp(i + 1, 0, n - 1) - origin, 0, span - 1);
	return a;
}

// bilinear mix of four fp32 texels (two packed halves each), exact sequence of bilin_mix()
struct Tex4
{
	f2 lo, hi; // (r, g), (b, a)
};
GRB_DEV Tex4 ld_tex(const float4 *p)
{
	float4 v = *p;
	Tex4 t;
	t.lo = make_float2(v.x, v.y);
	t.hi = make_float2(v.z, v.w);
	return t;
}
GRB_DEV f2 mix2(f2 t00, f2 t10, f2 t01, f2 t11, f2 a, f2 ia, f2 b, f2 ib)
{
	f2 top = add2(mul2(t00, ia), mul2(t10, a));
	f2 bot = add2(mul2(t01, ia), mul2(t11, a));
	return add2(mul2(top, ib), mul2(bot, b));
}

// 9-tap tent over an fp32 tile (row pitch `tw` texels): centre 1/4, then the tap order of tent9()
// in grb_post.cu -- (-,+) (0,+) (+,+) (-,0) (+,0) (-,-) (0,-) (+,-) -- accumulating acc += w * s
// with separate multiply and add.
GRB_DEV void tent9_tile(const float4 *tile, int tw, const Axis &xm, const Axis &xc, const Axis &xp, const Axis &ym, const Axis &yc, const Axis &yp, f2 &out_lo,
                        f2 &out_hi)
{
	f2 acc_lo, acc_hi;
	auto tap = [&](const Axis &ax, const Axis &ay, float weight, bool first) {
		const float4 *r0 = tile + ay.i0 * tw, *r1 = tile + ay.i1 * tw;
		Tex4 t00 = ld_tex(r0 + ax.i0), t10 = ld_tex(r0 + ax.i1), t01 = ld_tex(r1 + ax.i0), t11 = ld_tex(r1 + ax.i1);
		const f2 a = mk2(ax.w), ia = mk2(fsub(1.0f, ax.w)), b = mk2(ay.w), ib = mk2(fsub(1.0f, ay.w));
		f2 lo = mix2(t00.lo, t10.lo, t01.lo, t11.lo, a, ia, b, ib);
		f2 hi = mix2(t00.hi, t10.hi, t01.hi, t11.hi, a, ia, b, ib);
		if (first)
		{
			acc_lo = mul2(mk2(weight), lo);
			acc_hi = mul2(mk2(weight), hi);
		}
		else
		{
			acc_lo = add2(acc_lo, mul2(mk2(weight), lo));
			acc_hi = add2(acc_hi, mul2(mk2(weight), hi));
		}
	};
	tap(xc, yc, 0.25f, true);
	tap(xm, yp, 0.0625f, false);
	tap(xc, yp, 0.125f, false);
	tap(xp, yp, 0.0625f, false);
	tap(xm, yc, 0.125f, false);
	tap(xp, yc, 0.125f, false);
	tap(xm, ym, 0.0625f, false);
	tap(xc, ym, 0.125f, false);
	tap(xp, ym, 0.0625f, false);
	out_lo = acc_lo;
	out_hi = acc_hi;
}

GRB_DEV float4 widen(uint2 t)
{
	return unpack_rgba16f(t);
}

// ---------------------------------------------------------------------------------- K8 / K9 tiled
struct TentArgs
{
	View<uint2> out;
	View<const uint2> history; // Feedback only
	float lerp;
	int in_w, in_h;
	int y0, y1; // output rows
	float inv_w, inv_h, inv_in_w, inv_in_h;
};

template <bool Up, bool Feedback>
__global__ void __launch_bounds__(kThreads) tent_tile_kernel(const __grid_constant__ CUtensorMap src_map, const TentArgs a)
{
	constexpr int SW = Up ? kUpSrcW : kDownSrcW, SH = Up ? kUpSrcH : kDownSrcH;
	constexpr float kOff = Up ? 0.875f : 1.75f;
	extern __shared__ __align__(128) unsigned char smem[];
	uint2 *raw = reinterpret_cast<uint2 *>(smem);                                    // SW x SH texels, as landed
	float4 *tile = reinterpret_cast<float4 *>(smem + ((SW * SH * 8 + 127) & ~127)); // the same, fp32
	__shared__ __align__(8) uint64_t bar_storage;
	const uint32_t bar = smem_u32(&bar_storage);

	const int ox0 = blockIdx.x * kOutW, oy0 = a.y0 + blockIdx.y * kOutH;
	const int sx0 = Up ? (ox0 >> 1) - 2 : 2 * ox0 - 2;
	const int sy0 = Up ? (oy0 >> 1) - 2 : 2 * oy0 - 2; // oy0 - a.y0 is a multiple of 16; for Up an odd a.y0 only widens the margin by rounding down
	if (threadIdx.x == 0)
		mbar_init(bar);
	__syncthreads();
	if (threadIdx.x == 0)
		tma_load_box(smem_u32(raw), &src_map, sx0 * 2, sy0, bar, SW * SH * 8);
	mbar_wait(bar, 0);
	for (int i = threadIdx.x; i < SW * SH; i += kThreads)
	{
		const int ry = i / SW, rx = i - ry * SW;
		tile[ry * SW + col_slot<SW, !Up>(rx)] = widen(raw[i]);
	}
	__syncthreads();

	const int lx = threadIdx.x & (kOutW - 1);
	const int x = ox0 + lx;
#pragma unroll 1
	for (int ly = threadIdx.x / kOutW; ly < kOutH; ly += kThreads / kOutW)
	{
		const int y = oy0 + ly;
		if (x >= a.out.w || y >= a.y1)
			continue;
		const float u = ((float)x + 0.5f) * a.inv_w, v = ((float)y + 0.5f) * a.inv_h;
		const float du = kOff * a.inv_in_w, dv = kOff * a.inv_in_h;
		Axis xm = axis_setup(u + (-du), a.in_w, sx0, SW), xc = axis_setup(u, a.in_w, sx0, SW), xp = axis_setup(u + du, a.in_w, sx0, SW);
		const Axis ym = axis_setup(v + (-dv), a.in_h, sy0, SH), yc = axis_setup(v, a.in_h, sy0, SH), yp = axis_setup(v + dv, a.in_h, sy0, SH);
		xm.i0 = col_slot<SW, !Up>(xm.i0); xm.i1 = col_slot<SW, !Up>(xm.i1);
		xc.i0 = col_slot<SW, !Up>(xc.i0); xc.i1 = col_slot<SW, !Up>(xc.i1);
		xp.i0 = col_slot<SW, !Up>(xp.i0); xp.i1 = col_slot<SW, !Up>(xp.i1);
		f2 lo, hi;
		tent9_tile(tile, SW, xm, xc, xp, ym, yc, yp, lo, hi);
		float4 value = make_float4(lo.x, lo.y, hi.x, hi.y);
		if (Feedback)
		{
			float4 hs = unpack_rgba16f(__ldg(&a.history.at(x, y)));
			value = make_float4(fmix(hs.x, value.x, a.lerp), fmix(hs.y, value.y, a.lerp), fmix(hs.z, value.z, a.lerp), fmix(hs.w, value.w, 1.0f));
		}
		a.out.at(x, y) = pack_rgba16f(value);
	}
}

// ---------------------------------------------------------------------------------- K7 + K8 fused
// Row-sharded frames: the d0 band is stored into the 1/4-resolution image of EVERY rank (peer memory over
// NVLink / NVSwitch) and the last CTA publishes the frame's epoch in every rank's flag array
// (grb_peer.cuh).  peers.count == 0: plain local store to HeadArgs::d0.

struct HeadArgs
{
	View<uint2> d0;
	View<uint2> t; // optional (p == nullptr: the threshold image is not materialised)
	const float *lum;
	int hdr_w, hdr_h, t_w, t_h;
	int y0, y1; // d0 rows
	float inv_t_w, inv_t_h, inv_d0_w, inv_d0_h;
};

constexpr int kHeadHdrW = 2 * kDownSrcW, kHeadHdrH = 2 * kDownSrcH; // 136 x 72 HDR texels

struct AxisRec
{
	short i0, i1;
	float w;
};

template <bool DynamicExposure>
__global__ void __launch_bounds__(kThreads) bloom_head_kernel(const __grid_constant__ CUtensorMap hdr_map, const HeadArgs a, const PeerTargets peers)
{
	__builtin_assume(threadIdx.y == 0); // 1-D blocks: peer_publish's leader test is threadIdx.x == 0
	extern __shared__ __align__(128) unsigned char smem[];
	uint32_t *hdr = reinterpret_cast<uint32_t *>(smem);                                    // 136 x 72 B10G11R11
	float4 *tile = reinterpret_cast<float4 *>(smem + kHeadHdrW * kHeadHdrH * 4);           // 68 x 36 threshold texels, fp32 of their fp16 value
	AxisRec *colrec = reinterpret_cast<AxisRec *>(smem + kHeadHdrW * kHeadHdrH * 4 + kDownSrcW * kDownSrcH * 16);
	AxisRec *rowrec = colrec + kDownSrcW;
	__shared__ __align__(8) uint64_t bar_storage;
	const uint32_t bar = smem_u32(&bar_storage);

	const int ox0 = blockIdx.x * kOutW, oy0 = a.y0 + blockIdx.y * kOutH;
	const int tx0 = 2 * ox0 - 2, ty0 = 2 * oy0 - 2;
	const int hx0 = 2 * tx0, hy0 = 2 * ty0;
	if (threadIdx.x == 0)
		mbar_init(bar);
	__syncthreads();
	if (threadIdx.x == 0)
		tma_load_box(smem_u32(hdr), &hdr_map, hx0, hy0, bar, kHeadHdrW * kHeadHdrH * 4);
	// while the tile is in flight: the HDR footprint of every threshold column / row of the tile
	// (bloom_threshold.comp:28-30: one LinearClamp sample at the output texel centre)
	if (threadIdx.x < kDownSrcW + kDownSrcH)
	{
		const bool is_col = threadIdx.x < kDownSrcW;
		const int k = is_col ? threadIdx.x : threadIdx.x - kDownSrcW;
		const int t = (is_col ? tx0 : ty0) + k;
		const float c = ((float)t + 0.5f) * (is_col ? a.inv_t_w : a.inv_t_h);
		const Axis ax = axis_setup(c, is_col ? a.hdr_w : a.hdr_h, is_col ? hx0 : hy0, is_col ? kHeadHdrW : kHeadHdrH);
		AxisRec r;
		r.i0 = (short)ax.i0;
		r.i1 = (short)ax.i1;
		r.w = ax.w;
		(is_col ? colrec : rowrec)[k] = r;
	}
	const float lum_sub = DynamicExposure ? 8.0f * __ldg(&a.lum[1]) : 8.0f;
	__syncthreads();
	mbar_wait(bar, 0);

	// ---- threshold tile (bloom_threshold.comp:23-45), only texels that exist in the image ----
	for (int i = threadIdx.x; i < kDownSrcW * kDownSrcH; i += kThreads)
	{
		const int ly = i / kDownSrcW, lx = i - ly * kDownSrcW;
		const int tx = tx0 + lx, ty = ty0 + ly;
		if (tx < 0 || ty < 0 || tx >= a.t_w || ty >= a.t_h)
			continue;
		const AxisRec cx = colrec[lx], cy = rowrec[ly];
		const uint32_t *r0 = hdr + cy.i0 * kHeadHdrW, *r1 = hdr + cy.i1 * kHeadHdrW;
		const float3 t00 = unpack_r11g11b10(r0[cx.i0]), t10 = unpack_r11g11b10(r0[cx.i1]);
		const float3 t01 = unpack_r11g11b10(r1[cx.i0]), t11 = unpack_r11g11b10(r1[cx.i1]);
		// the sampler's weights (a, 1 - a, b, 1 - b), in lerp form
		const float wa = cx.w, wb = cy.w;
		float3 c;
		{
			const float tx = fmaf(wa, t10.x - t00.x, t00.x), bx = fmaf(wa, t11.x - t01.x, t01.x);
			const float ty = fmaf(wa, t10.y - t00.y, t00.y), by = fmaf(wa, t11.y - t01.y, t01.y);
			const float tz = fmaf(wa, t10.z - t00.z, t00.z), bz = fmaf(wa, t11.z - t01.z, t01.z);
			c = make_float3(fmaf(wb, bx - tx, tx), fmaf(wb, by - ty, ty), fmaf(wb, bz - tz, tz));
		}
		float luminance = fmax_(fmax_(c.x, c.y), c.z) + 0.0001f;
		// log2: the hardware approximation is good to ~2^-22 absolute, which is below half an fp16 ulp of
		// the stored value unless |log2| is tiny, i.e. luminance within ~1 % of 1
		const float loglum = fabsf(luminance - 1.0f) < 0.01f ? log2f(luminance) : lg2_fast(luminance);
		const float scale = (luminance - lum_sub) * rcp_fast(luminance);
		const uint2 packed = pack_rgba16f(make_float4(fmax_(c.x * scale, 0.0f), fmax_(c.y * scale, 0.0f), fmax_(c.z * scale, 0.0f), loglum));
		tile[ly * kDownSrcW + col_slot<kDownSrcW, true>(lx)] = unpack_rgba16f(packed); // what a sampler would read back from the RGBA16F image
		// the interior of the tile is this CTA's share of the threshold image
		if (a.t.p && lx >= 2 && lx < kDownSrcW - 2 && ly >= 2 && ly < kDownSrcH - 2 && ty >= 2 * a.y0 && ty < 2 * a.y1)
			a.t.at(tx, ty) = packed;
	}
	__syncthreads();

	// ---- 1/4-resolution downsample from the tile (bloom_downsample.comp:21-42) ----
	const int lx = threadIdx.x & (kOutW - 1);
	const int x = ox0 + lx;
#pragma unroll 1
	for (int ly = threadIdx.x / kOutW; ly < kOutH; ly += kThreads / kOutW)
	{
		const int y = oy0 + ly;
		if (x >= a.d0.w || y >= a.y1)
			continue;
		const float u = ((float)x + 0.5f) * a.inv_d0_w, v = ((float)y + 0.5f) * a.inv_d0_h;
		const float du = 1.75f * a.inv_t_w, dv = 1.75f * a.inv_t_h;
		Axis xm = axis_setup(u + (-du), a.t_w, tx0, kDownSrcW), xc = axis_setup(u, a.t_w, tx0, kDownSrcW), xp = axis_setup(u + du, a.t_w, tx0, kDownSrcW);
		const Axis ym = axis_setup(v + (-dv), a.t_h, ty0, kDownSrcH), yc = axis_setup(v, a.t_h, ty0, kDownSrcH), yp = axis_setup(v + dv, a.t_h, ty0, kDownSrcH);
		xm.i0 = col_slot<kDownSrcW, true>(xm.i0); xm.i1 = col_slot<kDownSrcW, true>(xm.i1);
		xc.i0 = col_slot<kDownSrcW, true>(xc.i0); xc.i1 = col_slot<kDownSrcW, true>(xc.i1);
		xp.i0 = col_slot<kDownSrcW, true>(xp.i0); xp.i1 = col_slot<kDownSrcW, true>(xp.i1);
		f2 lo, hi;
		tent9_tile(tile, kDownSrcW, xm, xc, xp, ym, yc, yp, lo, hi);
		const uint2 texel = pack_rgba16f(make_float4(lo.x, lo.y, hi.x, hi.y));
		if (peers.count == 0)
			a.d0.at(x, y) = texel;
		else
		{
			const size_t at = (size_t)y * a.d0.pitch + x;
			for (int r = 0; r < peers.count; r++)
				static_cast<uint2 *>(peers.data[r])[at] = texel;
		}
	}
	if (peers.count != 0)
		peer_publish(peers);
}

constexpr size_t tent_smem(bool up)
{
	return (size_t)(((up ? kUpSrcW * kUpSrcH : kDownSrcW * kDownSrcH) * 8 + 127) & ~127) + (size_t)(up ? kUpSrcW * kUpSrcH : kDownSrcW * kDownSrcH) * 16;
}
constexpr size_t kHeadSmem = (size_t)kHeadHdrW * kHeadHdrH * 4 + (size_t)kDownSrcW * kDownSrcH * 16 + (size_t)(kDownSrcW + kDownSrcH) * sizeof(AxisRec);

template <auto kernel> // one flag array per kernel (a function-pointer VALUE, not its type)
bool opt_in_smem(size_t bytes)
{
	// per device: the attribute belongs to the function in the current context
	static std::mutex lock;
	static bool done[64] = {};
	int device = 0;
	if (cudaGetDevice(&device) != cudaSuccess || device < 0 || device >= 64)
		return false;
	std::lock_guard<std::mutex> hold(lock);
	if (!done[device])
	{
		if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess)
		{
			cudaGetLastError();
			return false;
		}
		done[device] = true;
	}
	return true;
}

bool tiles_disabled()
{
	static const bool off = getenv("GRB_POST_NO_TILES") != nullptr;
	return off;
}
} // namespace

// Launchers used by the entry points in grb_post.cu.  Return false when the shape is not eligible
// (the caller then runs the generic kernel); true means "launched" and `*rc` holds the result.
bool launch_tent_tiled(bool up, const GrbImage *in, const GrbImage *history, float lerp, const GrbImage *out, GrbRows rows, cudaStream_t stream, int32_t *rc)
{
	// Only the large levels (1/4 resolution of a 4K frame) are worth a tile kernel; the levels below stay
	// on the bit-exact generic kernels, which is also what the fused tail (grb_bloom_tail) computes -- a
	// level's arithmetic must not depend on whether the caller fused the tail or a frame is row-sharded.
	if (tiles_disabled() || (long long)out->width * out->height < 200000)
		return false;
	const bool shape_ok = up ? (out->width == 2 * in->width && out->height == 2 * in->height) : (in->width == 2 * out->width && in->height == 2 * out->height);
	if (!shape_ok || (up && history))
		return false;
	CUtensorMap map;
	if (!make_map_u32(&map, in, 2, (up ? kUpSrcW : kDownSrcW) * 2, up ? kUpSrcH : kDownSrcH))
		return false;
	TentArgs a;
	a.out = view_of<uint2>(out);
	a.history = history ? view_of<const uint2>(history) : View<const uint2>{};
	a.lerp = lerp;
	a.in_w = in->width;
	a.in_h = in->height;
	a.y0 = rows.y0;
	a.y1 = rows.y1;
	a.inv_w = 1.0f / (float)out->width;   // hdr.cpp:178-181, 208-211
	a.inv_h = 1.0f / (float)out->height;
	a.inv_in_w = 1.0f / (float)in->width;
	a.inv_in_h = 1.0f / (float)in->height;
	dim3 grid((out->width + kOutW - 1) / kOutW, (rows.y1 - rows.y0 + kOutH - 1) / kOutH, 1);
	if (up)
	{
		if (!opt_in_smem<tent_tile_kernel<true, false>>(tent_smem(true)))
			return false;
		tent_tile_kernel<true, false><<<grid, kThreads, tent_smem(true), stream>>>(map, a);
	}
	else if (history)
	{
		if (!opt_in_smem<tent_tile_kernel<false, true>>(tent_smem(false)))
			return false;
		tent_tile_kernel<false, true><<<grid, kThreads, tent_smem(false), stream>>>(map, a);
	}
	else
	{
		if (!opt_in_smem<tent_tile_kernel<false, false>>(tent_smem(false)))
			return false;
		tent_tile_kernel<false, false><<<grid, kThreads, tent_smem(false), stream>>>(map, a);
	}
	*rc = check_launch(up ? "grb_bloom_upsample" : "grb_bloom_downsample");
	return true;
}
} // namespace grb

using namespace grb;

namespace
{
int32_t launch_head(const char *what, const GrbImage *hdr, const float *luminance, const GrbImage *threshold_out, const GrbImage *d0, GrbRows rows,
                    const PeerTargets &peers, void *stream)
{
	if (!image_ok(hdr, GRB_FORMAT_B10G11R11_UFLOAT_PACK32, 4) || !d0 || d0->format != GRB_FORMAT_R16G16B16A16_SFLOAT || d0->width <= 0 || d0->height <= 0 ||
	    (d0->row_pitch % 8) != 0 || (peers.count == 0 && !image_ok(d0, GRB_FORMAT_R16G16B16A16_SFLOAT, 8)) ||
	    (threshold_out && !image_ok(threshold_out, GRB_FORMAT_R16G16B16A16_SFLOAT, 8)))
	{
		set_last_error("grb_bloom_threshold_downsample: hdr must be B10G11R11_UFLOAT, threshold_out / d0 R16G16B16A16_SFLOAT");
		return GRB_ERR_UNSUPPORTED_FORMAT;
	}
	const int tw = (hdr->width + 1) / 2, th = (hdr->height + 1) / 2; // ceil rule, render_graph.cpp:3160-3171
	if (threshold_out && (threshold_out->width != tw || threshold_out->height != th))
	{
		set_last_error("grb_bloom_threshold_downsample: threshold_out must be ceil(hdr / 2)");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	rows = full_rows(rows, d0->height);
	const int row_count = rows.y1 > rows.y0 ? rows.y1 - rows.y0 : 0;
	if (row_count == 0 && peers.count == 0)
		return GRB_OK;
	CUtensorMap map;
	const bool eligible = !tiles_disabled() && hdr->width == 2 * tw && hdr->height == 2 * th && tw == 2 * d0->width && th == 2 * d0->height &&
	                      make_map_u32(&map, hdr, 1, kHeadHdrW, kHeadHdrH) &&
	                      (luminance ? opt_in_smem<bloom_head_kernel<true>>(kHeadSmem) : opt_in_smem<bloom_head_kernel<false>>(kHeadSmem));
	if (!eligible)
	{
		set_last_error("grb_bloom_threshold_downsample: needs exact 2:1 size steps and 16-byte aligned rows; use grb_bloom_threshold + grb_bloom_downsample");
		return GRB_ERR_UNSUPPORTED_FORMAT;
	}
	HeadArgs a;
	a.d0 = view_of<uint2>(d0);
	a.t = threshold_out ? view_of<uint2>(threshold_out) : View<uint2>{};
	a.lum = luminance;
	a.hdr_w = hdr->width;
	a.hdr_h = hdr->height;
	a.t_w = tw;
	a.t_h = th;
	a.y0 = rows.y0;
	a.y1 = rows.y0 + row_count;
	a.inv_t_w = 1.0f / (float)tw; // hdr.cpp:140-141
	a.inv_t_h = 1.0f / (float)th;
	a.inv_d0_w = 1.0f / (float)d0->width;
	a.inv_d0_h = 1.0f / (float)d0->height;
	const dim3 grid = peer_grid(row_count, dim3((d0->width + kOutW - 1) / kOutW, (row_count + kOutH - 1) / kOutH, 1));
	if (luminance)
		bloom_head_kernel<true><<<grid, kThreads, kHeadSmem, as_stream(stream)>>>(map, a, peers);
	else
		bloom_head_kernel<false><<<grid, kThreads, kHeadSmem, as_stream(stream)>>>(map, a, peers);
	return check_launch(what);
}
} // namespace

// bloom_threshold.comp + the first bloom_downsample.comp dispatch in one pass (hdr.cpp:115-187):
// d0 = downsample(threshold(hdr)).  `threshold_out` may be NULL; when given, the rows of the
// threshold image that belong to d0's rows [rows.y0, rows.y1) -- threshold rows 2*y0 .. 2*y1 -- are
// written as well.
extern "C" int32_t grb_bloom_threshold_downsample(const GrbImage *hdr, const float *luminance, const GrbImage *threshold_out, const GrbImage *d0, GrbRows rows,
                                                  void *stream)
{
	PeerTargets none{};
	return launch_head("grb_bloom_threshold_downsample", hdr, luminance, threshold_out, d0, rows, none, stream);
}

// The same pass for a row-sharded frame: the band's d0 texels go to every rank's image and the
// flags are raised, exactly as grb_bloom_downsample_to_peers does for the unfused pair.
extern "C" int32_t grb_bloom_threshold_downsample_to_peers(const GrbImage *hdr, const float *luminance, const GrbImage *d0_layout, void *const *peer_images,
                                                           uint32_t *const *peer_flags, int32_t peer_count, int32_t flag_index, uint32_t epoch,
                                                           uint32_t *scratch_counter, GrbRows rows, void *stream)
{
	if (!d0_layout)
	{
		set_last_error("grb_bloom_threshold_downsample_to_peers: null d0_layout");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	PeerTargets peers;
	if (!peer_targets_from("grb_bloom_threshold_downsample_to_peers", peer_images, peer_flags, peer_count, flag_index, epoch, scratch_counter, peers))
		return GRB_ERR_INVALID_ARGUMENT;
	return launch_head("grb_bloom_threshold_downsample_to_peers", hdr, luminance, nullptr, d0_layout, rows, peers, stream);
}
