// shard_plan.hpp -- which rows of which image one rank of a row-sharded frame computes.
//
// Derived backwards from the rows a rank OWNS (its band of the backbuffer): every stage computes
// exactly the rows its consumers on this rank read, so nothing is missing at band edges and the
// sharded frame is bit-identical to the unsharded one.  Stencil reaches used:
//   FXAA      : +-1 px diagonal taps, direction taps <= 8 px * 0.5 + bilinear  -> 6 rows of tonemapped
//   tonemap   : bloom tap = bilinear of upsample-0 at (y+0.5)/4                 -> u0 rows y/4 -+ 1
//   d0 (1/4)  : 9-tap tent, +-1.75 texels of threshold around 2y+1 + bilinear   -> t rows 2y-2 .. 2y+3
//   threshold : bilinear of HDR at 2y+1                                         -> HDR rows 2y .. 2y+1 (+-1)
// Bands are aligned to 64 full-res rows, so the 1/4-res d0 bands tile that level exactly.
//
// SMAA 1x (grb_smaa.cu), preset with s = max_search_steps (4 / 8 / 16 / 32 for Low .. Ultra).  Every sample is a
// bilinear tap of a coordinate computed in fp32.  A tap whose nominal position is a texel centre (an integer row
// offset) can, after rounding, land a few ulp off it and then takes the neighbouring row with a weight of rounding
// size; such a row is counted below ("guard row"): in a sharded frame it would otherwise hold another frame's or
// another rank's bytes, and a weight of 1e-7 can still flip a tie or an 8-bit rounding.  Taps at quarter-row
// offsets (the searches) read exactly the two rows around them.
//   blend     : weights at +0 and +1 row (the .w / .y taps of the pixel to the right / below), colour at +-1 row
//               -> weights rows y-1 .. y+2, colour rows y-2 .. y+2 (guard rows included)
//   weights   : vertical edge, up search: taps at y - 1/4 - 2k, k = 0 .. s (the end test compares the accumulated
//               coordinate with one computed in one step, so rounding can allow one step more than s)
//               -> rows down to y-1-2s; the end tap (1.25 .. 3.25 rows back, integer for the lookup texture's values)
//               and the corner taps there -> y-2-2s with its guard row.
//               down search: taps at y + 5/4 + 2k -> rows up to y+2+2s; end tap + 1 row and corner taps
//               -> y+3+2s, y+4+2s with its guard row.
//               horizontal edge (+-2 rows with corners) and diagonal searches (<= 16 + 3 rows, High / Ultra only)
//               reach less.  -> edge rows y - (2s+2) .. y + (2s+4)
//   edges     : L at -2 .. +1 rows (Ltoptop, Lbottom)           -> colour rows y-3 .. y+2 (guard rows included)
// So a rank that owns rows [y0, y1) produces the edges of [y0, y1) only; its weight pass runs on [y0-1, y1+2) and
// reads the edge window [y0-2s-3, y1+2s+6), which the ranks owning those rows deliver (grb_smaa_edge_detection_to_peers);
// blend writes [y0, y1); the tonemap covers [y0-3, y1+2).  All clamped to the image (taps clamp to the edge rows).
//
// TAA (taa_kernel, grb_post.cu) sits between the lighting and the post chain: its colour output "HDR-resolved" is
// what the threshold and the tonemap read, so the TAA rows are the rows the lighting pass computes without TAA (the
// union of the tonemap rows and the threshold's HDR rows above, for the same FXAA / SMAA settings).  A TAA texel reads
//   current   : HDR at integer offsets -1 .. +1 in x and y (exact texel fetches, clamped to the image)
//   velocity  : depth and mv at integer offsets -1 .. +1 (the nearest-depth footprint, exact fetches)
//   history   : last frame's history at uv - mv (or at the reprojected position when mv = 0): any row, since the
//               motion vectors are an input -- not a halo: every rank holds the WHOLE history, assembled from every
//               rank's own rows of the last frame (grb_taa_resolve_to_peers, or an all-gather without peer memory).
// No fp32 coordinate takes part in the first two, so no guard row: lighting = TAA rows +-1, clamped.  Each rank
// produces the history of its own rows only; the TAA rows outside them are computed for the colour alone.
//
// FSR 1 (grb_fsr.cu) after the post chain: everything above runs at the render size (Wr x Hr), the two FSR passes
// write the display size (Wd x Hd), and the bands are display rows.  Two row sets then differ:
//   B (own)        the display band: what the rank owns and reads back.
//   P (render_own) the render rows the rank PRODUCES for the exchanges (the d0 push, the SMAA edge push, the TAA
//                  history push) and the bands of their NCCL all-gathers.  The interior boundary at display row y is
//                  8 * floor(y * Hr / (8 * Hd)), with 0 and Hr at the two ends; every rank computes every rank's P
//                  from the same inputs, so the ranks' P tile [0, Hr).  A layout in which some P is empty is refused.
// Derived backwards from B:
//   RCAS      : exact texel fetches at +-1 row (fsr_rcas_kernel)           -> RCAS rows B, EASU rows E = B +- 1
//               (without RCAS, E = B)
//   EASU      : output row y reads render rows around (y + 0.5) Hr / Hd - 0.5: ppy = y k1 + k3, fpy = floor(ppy),
//               p0y = fpy k5 + k7, and four gathers at p0y, p0y + k9, p0y + k11, p0y + k13 (constants of
//               grb_fsr_easu_constants); each gather's origin is floor(v Hr - 0.5), clamped to [-2, Hr + 1], and
//               unorm_texel clamps the row to the edge.  Gather 0 uses only the row after its origin (b, c), gathers
//               1 and 2 use both rows, gather 3 only its origin row (n, o).  The window W is the hull of those rows
//               over every y in E, computed on the host with the kernel's own fp32 operations (the host library is
//               built with -ffp-contract=off, the kernel with -fmad=false), so it is exact: no guard row.
//   final render-resolution image (FXAA output, SMAA blend, or the tonemap without AA) -> W
//   FXAA      : rows W with the first one rounded down to a multiple of 16, tonemap those +- 6.  The tile kernel
//               (fxaa_fast_kernel) runs 16-row tiles from its first row and forms its bilinear coordinates in fp32
//               relative to the tile, so a pixel's result depends on its offset in the tile: the tiles must start
//               on the rows they start on unsharded.  Without FSR the FXAA rows stay the band, as before (a band
//               that does not start on a multiple of 16 rows meets the same dependence there).
//   SMAA      : blend on W, weights W-1 .. W+2, the edge window from the weights as above; edges produced on P;
//               tonemap = hull of the blend's colour reads W-2 .. W+2 and the edge pass's P-3 .. P+2
//   upsample0, TAA and lighting rows follow from the tonemap as above; downsample0, threshold and the luminance grid
//   follow from P and Hr; the TAA rows also cover P, whose history the rank pushes.
// Without FSR, W = E = P = B, and every row above is what it is without this paragraph.
#pragma once

#include <vector>

#include "../../include/granite_b200.h"

namespace Granite
{
struct ShardPlan
{
	GrbRows own;        // backbuffer rows this rank owns (and reads back)
	GrbRows fxaa;       // rows of the FXAA output
	GrbRows tonemap;    // rows of "tonemapped"
	GrbRows upsample0;  // rows of "upsample-0" (1/4)
	GrbRows downsample0; // rows of "downsample-0" (1/4): this rank's contribution to the all-gather
	GrbRows threshold;  // rows of "threshold" (1/2)
	GrbRows taa;        // rows of "HDR-resolved" the TAA resolve computes (its history: the own rows)
	GrbRows lighting;   // rows of "HDR-main" (= rows of the G-buffer that must be resident)
	GrbRows lum_grid;   // rows of the (d3/2) luminance grid this rank samples
	// SMAA (smaa_quality >= 0); whole images when unsharded or without SMAA
	GrbRows smaa_blend;       // rows of the SMAA output (= own)
	GrbRows smaa_weights;     // rows of "smaa-weights" the blend reads
	GrbRows smaa_edges;       // rows of "smaa-edge" this rank produces (= own)
	GrbRows smaa_edge_window; // rows of "smaa-edge" the weight pass reads: delivered by the ranks that own them
	// FSR 1 upscaling; without it easu = own and easu_window = render_own = own
	GrbRows easu;        // display rows of the EASU output (own, +-1 with RCAS)
	GrbRows easu_window; // render rows EASU reads for them: the rows of the final render-resolution image
	GrbRows render_own;  // render rows this rank produces for the d0, SMAA edge and TAA history exchanges
};

// FSR 1 after the post chain: the render size the chain runs at (height 0: no upscale) and whether RCAS follows EASU.
struct ShardUpscale
{
	unsigned width = 0, height = 0;
	bool rcas = false;
};

// width x height: the display size the bands cut.  smaa_quality: SMAA preset 0..3 (Low .. Ultra) downstream of the
// tonemap, -1 for none.  taa: a TAA resolve between the lighting and the post chain (it widens the lighting rows).
// upscale: FSR 1 from the render size to the display size; throws std::invalid_argument when a rank's render rows
// (render_own) would be empty.
ShardPlan compute_shard_plan(unsigned width, unsigned height, const std::vector<GrbRows> &bands, unsigned rank, bool fxaa, int smaa_quality = -1,
                             bool taa = false, ShardUpscale upscale = {});

// Lighting in stripes (opt-in): rank r of W lights the stripes k with k mod W == r, rows [k s, min((k + 1) s, H)) for
// stripes of s rows, whatever the bands; the bands still decide who runs the post chain on which rows (the plan above,
// unchanged).  A rank then holds the HDR rows of its lighting rows L_r that it lit itself and receives the others from
// the ranks that lit them.  Lighting is per pixel and a light that cannot reach a pixel adds exactly 0, so any split of
// the rows gives the unsharded image bit for bit.
struct StripePlan
{
	std::vector<GrbRows> lit;               // S_r: this rank's stripes, clipped to the image
	std::vector<std::vector<GrbRows>> push; // [q]: the rows of S_r inside rank q's lighting rows L_q (none for q = rank)
	std::vector<GrbRows> receive;           // the rows of L_r that other ranks light
	std::vector<GrbRows> upload;            // S_r u L_r, merged: the G-buffer rows that must be resident
	std::vector<GrbRows> tile_rows;         // cluster tile-row ranges the lighting of S_r reads (cluster_tile_rows per stripe, merged)
};

// The stripe plan of `rank` for stripes of stripe_rows rows (a positive multiple of 8) with the same bands and post
// chain as compute_shard_plan, and a light cluster of cluster_rows tile rows.  Unsharded (one band): the whole image.
// Throws std::invalid_argument for a bad stripe height.
StripePlan compute_stripe_plan(unsigned width, unsigned height, const std::vector<GrbRows> &bands, unsigned rank, bool fxaa, int smaa_quality,
                               bool taa, unsigned stripe_rows, unsigned cluster_rows);

// The cluster tile rows under pixel rows [y0, y1) of a frame `height` rows tall with `resolution_y` tile rows: a tile
// row of a pixel row is floor((y + 0.5) / height * resolution_y) (clustering.frag through clusterer_bindless.h:29-40);
// one tile row of margin either side covers the rounding of that product.
GrbRows cluster_tile_rows(int y0, int y1, int height, int resolution_y);

// A new layout for moving the cuts of a sharded frame: throws std::invalid_argument unless `bands` tile [0, height) in
// order, or (under FSR 1) when a rank would produce no render rows.
void check_band_layout(unsigned width, unsigned height, const std::vector<GrbRows> &bands, ShardUpscale upscale);
} // namespace Granite
