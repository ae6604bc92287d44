#include "shard_plan.hpp"

#include <algorithm>
#include <cmath>
#include <stdexcept>
#include <string>

namespace Granite
{
namespace
{
unsigned ceil_scale(unsigned v, float s) { return (unsigned)std::max(1.0f, std::ceil(v * s)); }

GrbRows clamp_rows(int y0, int y1, unsigned h)
{
	GrbRows r;
	r.y0 = std::max(y0, 0);
	r.y1 = std::min(y1, (int)h);
	if (r.y1 <= r.y0)
		r.y1 = r.y0 + 1;
	return r;
}

GrbRows scale_band(GrbRows band, unsigned from_h, unsigned to_h)
{
	GrbRows r;
	r.y0 = (int)(((uint64_t)band.y0 * to_h) / from_h);
	r.y1 = (int)(((uint64_t)band.y1 * to_h + from_h - 1) / from_h);
	return r;
}

// First render row rank r produces: 8 * floor(y * Hr / (8 * Hd)) for its band's first display row y.
int render_cut(const std::vector<GrbRows> &bands, unsigned r, unsigned height, unsigned render_height)
{
	if (r == 0)
		return 0;
	if (r >= bands.size())
		return (int)render_height;
	return (int)(8 * (((uint64_t)bands[r].y0 * render_height) / (8 * (uint64_t)height)));
}

// Render rows fsr_easu_kernel reads for the display rows `rows` (derivation in shard_plan.hpp).
GrbRows easu_window(GrbRows rows, unsigned width, unsigned height, ShardUpscale up)
{
	float k[16];
	grb_fsr_easu_constants((int32_t)up.width, (int32_t)up.height, (int32_t)width, (int32_t)height, k);
	const int hr = (int)up.height;
	auto origin = [&](float v) {
		float f = std::floor(v * (float)hr - 0.5f);
		f = std::fmin(std::fmax(f, -2.0f), (float)hr + 1.0f);
		return (int)f;
	};
	int lo = hr, hi = -1;
	auto add = [&](int row) {
		row = std::min(std::max(row, 0), hr - 1);
		lo = std::min(lo, row);
		hi = std::max(hi, row);
	};
	for (int y = rows.y0; y < rows.y1; y++)
	{
		const float ppy = (float)y * k[1] + k[3];
		const float fpy = std::floor(ppy);
		const float p0y = fpy * k[5] + k[7];
		const int o0 = origin(p0y), o1 = origin(p0y + k[9]), o2 = origin(p0y + k[11]), o3 = origin(p0y + k[13]);
		add(o0 + 1);
		add(o1);
		add(o1 + 1);
		add(o2);
		add(o2 + 1);
		add(o3);
	}
	return GrbRows{ lo, hi + 1 };
}
} // namespace

ShardPlan compute_shard_plan(unsigned width, unsigned height, const std::vector<GrbRows> &bands, unsigned rank, bool fxaa, int smaa_quality, bool taa,
                             ShardUpscale upscale)
{
	ShardPlan p = {};
	const bool fsr = upscale.height > 0;
	const unsigned hr = fsr ? upscale.height : height; // rows of every image before the FSR passes
	const GrbRows whole = { 0, (int)hr };
	p.smaa_blend = p.smaa_weights = p.smaa_edges = p.smaa_edge_window = whole;
	const unsigned h_half = ceil_scale(hr, 0.5f), h_quarter = ceil_scale(hr, 0.25f);
	const unsigned h_d3 = ceil_scale(hr, 0.03125f), h_grid = h_d3 / 2;
	if (bands.size() <= 1)
	{
		p.own = p.easu = GrbRows{ 0, (int)height };
		p.fxaa = p.tonemap = p.taa = p.lighting = p.easu_window = p.render_own = whole;
		p.upsample0 = p.downsample0 = GrbRows{ 0, (int)h_quarter };
		p.threshold = GrbRows{ 0, (int)h_half };
		p.lum_grid = GrbRows{ 0, (int)h_grid };
		return p;
	}
	p.own = bands[rank];
	if (fsr)
	{
		// derivation in shard_plan.hpp
		for (unsigned r = 0; r < bands.size(); r++)
			if (render_cut(bands, r + 1, height, hr) <= render_cut(bands, r, height, hr))
				throw std::invalid_argument("FSR 1 upscaling from " + std::to_string(hr) + " to " + std::to_string(height) + " rows: rank " +
				                            std::to_string(r) + "'s band [" + std::to_string(bands[r].y0) + ", " + std::to_string(bands[r].y1) +
				                            ") produces no render rows (its borders fall into one 8-row unit of the render image); use wider bands");
		p.render_own = GrbRows{ render_cut(bands, rank, height, hr), render_cut(bands, rank + 1, height, hr) };
		p.easu = upscale.rcas ? clamp_rows(p.own.y0 - 1, p.own.y1 + 1, height) : p.own;
		p.easu_window = easu_window(p.easu, width, height, upscale);
	}
	else
		p.render_own = p.easu = p.easu_window = p.own;
	const GrbRows fin = p.easu_window, prod = p.render_own; // final render-resolution rows, produced rows
	p.fxaa = fin;
	if (fsr)
		p.fxaa.y0 &= ~15; // the FXAA tile kernel's 16-row tiles sit where they sit unsharded (shard_plan.hpp)
	p.tonemap = fxaa ? clamp_rows(p.fxaa.y0 - 6, p.fxaa.y1 + 6, hr) : fin;
	if (smaa_quality >= 0)
	{
		// derivation in shard_plan.hpp
		const int steps = 4 << std::min(smaa_quality, 3);
		p.smaa_blend = fin;
		p.smaa_edges = prod;
		p.smaa_weights = clamp_rows(fin.y0 - 1, fin.y1 + 2, hr);
		p.smaa_edge_window = clamp_rows(p.smaa_weights.y0 - (2 * steps + 2), p.smaa_weights.y1 + 2 * steps + 4, hr);
		p.tonemap = clamp_rows(std::min(fin.y0 - 2, prod.y0 - 3), std::max(fin.y1 + 2, prod.y1 + 2), hr);
	}
	p.upsample0 = clamp_rows(p.tonemap.y0 / 4 - 1, (p.tonemap.y1 + 3) / 4 + 1, h_quarter);
	p.downsample0 = scale_band(prod, hr, h_quarter);
	p.threshold = clamp_rows(2 * p.downsample0.y0 - 2, 2 * p.downsample0.y1 + 2, h_half);
	GrbRows hdr_for_threshold = clamp_rows(2 * p.threshold.y0 - 1, 2 * p.threshold.y1 + 1, hr);
	// the TAA rows also cover the produced rows, whose history this rank pushes (without FSR the tonemap holds them)
	p.taa = clamp_rows(std::min({ p.tonemap.y0, hdr_for_threshold.y0, prod.y0 }), std::max({ p.tonemap.y1, hdr_for_threshold.y1, prod.y1 }), hr);
	// TAA reads HDR, depth and mv at integer offsets of +-1 row (derivation in shard_plan.hpp)
	p.lighting = taa ? clamp_rows(p.taa.y0 - 1, p.taa.y1 + 1, hr) : p.taa;
	// luminance grid rows: row g belongs to the rank whose produced rows hold the first render row it maps to
	auto begin_of = [&](unsigned r) {
		const int y0 = fsr ? render_cut(bands, r, height, hr) : bands[r].y0;
		return (int)(((uint64_t)y0 * h_grid + hr - 1) / hr);
	};
	p.lum_grid.y0 = begin_of(rank);
	p.lum_grid.y1 = rank + 1 < bands.size() ? begin_of(rank + 1) : (int)h_grid;
	return p;
}

namespace
{
// The ranges of `rows` (in increasing order of y0) with overlapping or touching ones merged.
std::vector<GrbRows> merged(std::vector<GrbRows> rows)
{
	std::sort(rows.begin(), rows.end(), [](const GrbRows &a, const GrbRows &b) { return a.y0 < b.y0; });
	std::vector<GrbRows> out;
	for (const GrbRows &r : rows)
	{
		if (r.y1 <= r.y0)
			continue;
		if (!out.empty() && r.y0 <= out.back().y1)
			out.back().y1 = std::max(out.back().y1, r.y1);
		else
			out.push_back(r);
	}
	return out;
}

// The rows of `set` (disjoint ranges in increasing order) inside `with`.
std::vector<GrbRows> intersect(const std::vector<GrbRows> &set, GrbRows with)
{
	std::vector<GrbRows> out;
	for (const GrbRows &r : set)
	{
		const int y0 = std::max(r.y0, with.y0), y1 = std::min(r.y1, with.y1);
		if (y1 > y0)
			out.push_back(GrbRows{ y0, y1 });
	}
	return out;
}
} // namespace

GrbRows cluster_tile_rows(int y0, int y1, int height, int resolution_y)
{
	int t0 = int((long long)y0 * (long long)resolution_y / height) - 1;
	int t1 = int(((long long)y1 * (long long)resolution_y + height - 1) / height) + 1;
	return GrbRows{ std::max(t0, 0), std::min(t1, resolution_y) };
}

StripePlan compute_stripe_plan(unsigned width, unsigned height, const std::vector<GrbRows> &bands, unsigned rank, bool fxaa, int smaa_quality,
                               bool taa, unsigned stripe_rows, unsigned cluster_rows)
{
	if (stripe_rows == 0 || stripe_rows % 8 != 0)
		throw std::invalid_argument("lighting stripes must be a positive multiple of 8 rows (got " + std::to_string(stripe_rows) + ")");
	StripePlan sp;
	const unsigned world = std::max<unsigned>((unsigned)bands.size(), 1u);
	for (unsigned y = rank * stripe_rows; y < height; y += world * stripe_rows)
		sp.lit.push_back(GrbRows{ (int)y, (int)std::min(y + stripe_rows, height) });
	sp.push.resize(world);
	const GrbRows own_lighting = compute_shard_plan(width, height, bands, rank, fxaa, smaa_quality, taa).lighting;
	if (world > 1)
		for (unsigned q = 0; q < world; q++)
			if (q != rank)
				sp.push[q] = intersect(sp.lit, compute_shard_plan(width, height, bands, q, fxaa, smaa_quality, taa).lighting);
	// L_r minus S_r
	int y = own_lighting.y0;
	for (const GrbRows &r : intersect(sp.lit, own_lighting))
	{
		if (r.y0 > y)
			sp.receive.push_back(GrbRows{ y, r.y0 });
		y = r.y1;
	}
	if (y < own_lighting.y1)
		sp.receive.push_back(GrbRows{ y, own_lighting.y1 });
	std::vector<GrbRows> all = sp.lit;
	all.push_back(own_lighting);
	sp.upload = merged(all);
	std::vector<GrbRows> tiles;
	for (const GrbRows &r : sp.lit)
		tiles.push_back(cluster_tile_rows(r.y0, r.y1, (int)height, (int)cluster_rows));
	sp.tile_rows = merged(tiles);
	return sp;
}

void check_band_layout(unsigned width, unsigned height, const std::vector<GrbRows> &bands, ShardUpscale upscale)
{
	int expect = 0;
	for (const GrbRows &b : bands)
	{
		if (b.y0 != expect || b.y1 <= b.y0)
			throw std::invalid_argument("the bands must tile the frame in order");
		expect = b.y1;
	}
	if (expect != (int)height)
		throw std::invalid_argument("the bands must cover rows [0, " + std::to_string(height) + ")");
	if (upscale.height && bands.size() > 1)
		compute_shard_plan(width, height, bands, 0, false, -1, false, upscale); // throws when a rank would produce no render rows
}
} // namespace Granite
