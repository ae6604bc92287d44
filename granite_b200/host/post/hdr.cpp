// hdr.cpp -- "bloom-compute" + "tonemap" pass builders (renderer/post/hdr.cpp:35-400), recording
// C-ABI kernel launches on the graph's CUDA stream instead of Vulkan dispatches.  Push-constant
// values (inverse sizes, lerp factors) are computed by the kernels' launchers exactly as the
// reference's builders compute them; the formulas that live on this side are the frame-time
// dependent ones.
//
// Row-sharded frames: levels t (1/2) and d0 (1/4) -- 95 % of the bloom bytes -- are produced for
// the rank's own band only; d0 bands are exchanged (peer stores from the downsample kernel, or
// NCCL broadcasts), the pyramid tail (d1..d3, u2, u1: < 1.5 MB
// in total at 4K) is computed redundantly on every rank, the average-luminance grid is summed
// across ranks, u0 and the tonemap are again band-only.  Every texel any rank computes is
// computed from the same inputs by the same kernel, so the frame is bit-identical for any
// number of ranks.
#include "hdr.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <memory>
#include <utility>

namespace Granite
{
namespace
{
struct BloomResources
{
	RenderTextureResource *t, *d0, *u0, *d1, *u1, *d2, *u2, *d3, *hdr;
	const RenderBufferResource *lum;
	const RenderBufferResource *lum_grid;
};

GrbRows all_rows() { return GrbRows{ 0, 0 }; }

void bloom_build_compute(Vulkan::CommandBuffer &cmd, RenderGraph &graph, const FrameParameters &frame, const BloomResources &r)
{
	void *stream = cmd.get_stream_handle();
	auto img = [&](RenderTextureResource *res) { return graph.get_physical_texture_resource(*res).as_grb(); };
	float *lum = r.lum ? graph.get_physical_buffer_resource(*r.lum).get<float>() : nullptr;

	GrbImage hdr = img(r.hdr), t = img(r.t), d0 = img(r.d0), d1 = img(r.d1), d2 = img(r.d2), d3 = img(r.d3);
	GrbImage u2 = img(r.u2), u1 = img(r.u1), u0 = img(r.u0);
	const bool sharded = graph.is_sharded() && graph.get_shard_count() > 1;

	// Rows of each band-only level (shard_plan.hpp derives them from the rows this rank owns).
	const ShardPlan plan = graph.get_shard_plan();
	GrbRows d0_rows = sharded ? plan.downsample0 : all_rows();
	GrbRows t_rows = sharded ? plan.threshold : all_rows();

	// bloom_threshold_build_compute + the first bloom_downsample_build_compute (hdr.cpp:355-356), which
	// use LAST frame's average luminance.  Preferred form: ONE kernel with the threshold image kept in
	// shared memory (grb_bloom_threshold_downsample*); the threshold image is only written out when
	// GRB_BLOOM_KEEP_THRESHOLD is set (nothing downstream reads it).  Row-sharded frames need the d0
	// bands in full on every rank: the same kernel stores its band into every rank's copy over NVLink
	// peer memory and raises a flag (no collective launch, no second pass over the band); otherwise NCCL
	// broadcasts after a local pass.  The unfused pair remains for shapes the tile kernel does not cover.
	const bool keep_threshold = getenv("GRB_BLOOM_KEEP_THRESHOLD") != nullptr;
	RenderGraphCollectives::PeerSlot slot;
	const bool peer_stores = sharded && graph.get_collectives()->peer_exchange_begin_frame(RenderGraphCollectives::PeerChannel::BloomD0,
	                                                                                       (size_t)d0.row_pitch * (size_t)d0.height, slot);
	if (peer_stores)
	{
		const unsigned self = graph.get_collectives()->get_rank();
		int32_t rc = grb_bloom_threshold_downsample_to_peers(&hdr, lum, &d0, slot.images, slot.flags, (int32_t)slot.count, (int32_t)self, slot.epoch,
		                                                     slot.counter, d0_rows, stream);
		if (rc == GRB_ERR_UNSUPPORTED_FORMAT)
		{
			cmd.check(grb_bloom_threshold(&hdr, lum, &t, t_rows, stream), "grb_bloom_threshold");
			rc = grb_bloom_downsample_to_peers(&t, &d0, slot.images, slot.flags, (int32_t)slot.count, (int32_t)self, slot.epoch, slot.counter, d0_rows, stream);
		}
		cmd.check(rc, "grb_bloom_downsample_to_peers");
		d0.data = slot.images[self]; // the pyramid tail reads the exchanged copy
	}
	else if (grb_bloom_threshold_downsample(&hdr, lum, keep_threshold ? &t : nullptr, &d0, d0_rows, stream) != GRB_OK)
	{
		cmd.check(grb_bloom_threshold(&hdr, lum, &t, t_rows, stream), "grb_bloom_threshold");
		cmd.check(grb_bloom_downsample(&t, nullptr, 0.0f, &d0, d0_rows, stream), "grb_bloom_downsample(d0)");
	}
	// Everything above wants the whole machine for a few tens of microseconds; everything below is latency-bound
	// and small.  The next frame's lighting pass (a persistent kernel that takes every SM it is given) waits for this
	// mark, so the two do not fight over SMs, and starts while the pyramid tail below -- already resident on a
	// few SMs, see max_ctas -- runs beside it.
	graph.signal_mark("bloom-head", cmd);

	if (sharded && !peer_stores)
		graph.get_collectives()->all_gather_rows(cmd, graph.get_physical_texture_resource(*r.d0), graph.get_shard_plan_rows(&ShardPlan::downsample0));

	// d3 blends with its own previous frame (hdr.cpp:156-167, 182): lerp = 1 - 0.001^frame_time;
	// luminance_build_compute (hdr.cpp:68-98): size = d3 / 2, lerp = 1 - 0.5^frame_time, clamp [-3, 2]
	auto *history = graph.get_physical_history_texture_resource(*r.d3);
	GrbImage hist;
	if (history)
		hist = history->as_grb();
	const float lerp_d3 = float(1.0 - std::pow(0.001, frame.frame_time));
	const float lerp_lum = float(1.0 - std::pow(0.5, frame.frame_time));
	// with the exchanged d0 every rank holds the whole d3 and reduces it locally; the NCCL path keeps
	// the reference split (band partial sums + all-reduce, SURVEY.md section 8e) and the separate calls
	const bool nccl_luminance = lum && sharded && r.lum_grid && !peer_stores;

	// Everything below 1/4 resolution -- d1, d2, d3, luminance, u2, u1 -- and the last upsample u0 (own band + the
	// tonemap halo when row-sharded) is one cooperative launch (grid barriers between the levels); separate
	// dispatches when that is not available.  Row-sharded frames: the kernel itself waits for the peers' d0 bands.
	GrbRows u0_rows = sharded ? plan.upsample0 : all_rows();
	bool tail_fused = false, peers_awaited = false;
	if (!nccl_luminance)
	{
		static const int tail_ctas = [] {
			const char *e = getenv("GRB_BLOOM_TAIL_CTAS");
			return e ? atoi(e) : 16;
		}();
		GrbBloomTailOptions opt = {};
		opt.u0 = &u0;
		opt.u0_rows = u0_rows;
		if (peer_stores)
		{
			opt.peer_flags = slot.flags[graph.get_collectives()->get_rank()];
			opt.peer_count = (int32_t)slot.count;
			opt.peer_epoch = slot.epoch;
		}
		opt.max_ctas = tail_ctas;
		tail_fused = grb_bloom_tail_ex(&d0, &d1, &d2, &d3, history ? &hist : nullptr, lerp_d3, lum, lerp_lum, -3.0f, 2.0f, &u2, &u1, &opt, stream) == GRB_OK;
		peers_awaited = tail_fused;
	}
	if (peer_stores && !peers_awaited)
		cmd.check(grb_peer_wait(slot.flags[graph.get_collectives()->get_rank()], (int32_t)slot.count, slot.epoch, stream), "grb_peer_wait");
	if (!tail_fused)
	{
		cmd.check(grb_bloom_downsample(&d0, nullptr, 0.0f, &d1, all_rows(), stream), "grb_bloom_downsample(d1)");
		cmd.check(grb_bloom_downsample(&d1, nullptr, 0.0f, &d2, all_rows(), stream), "grb_bloom_downsample(d2)");
		cmd.check(grb_bloom_downsample(&d2, history ? &hist : nullptr, lerp_d3, &d3, all_rows(), stream), "grb_bloom_downsample(d3)");
		if (nccl_luminance)
		{
			// each rank samples the grid rows of its own band; the sum over ranks of (value or 0)
			// reassembles the grid exactly, then every rank reduces it in the shader's order
			float *grid = graph.get_physical_buffer_resource(*r.lum_grid).get<float>();
			const int size_x = d3.width / 2, size_y = d3.height / 2;
			Vulkan::cuda_ok(cudaMemsetAsync(grid, 0, sizeof(float) * size_x * size_y, reinterpret_cast<cudaStream_t>(cmd.get_stream())),
			                "cudaMemsetAsync(luminance grid)");
			GrbRows grid_rows = plan.lum_grid;
			if (grid_rows.y1 > grid_rows.y0)
				cmd.check(grb_luminance_grid(&d3, grid, grid_rows, stream), "grb_luminance_grid");
			graph.get_collectives()->all_reduce_sum(cmd, grid, (size_t)size_x * size_y);
			cmd.check(grb_luminance_finalize(grid, size_x, size_y, lum, lerp_lum, -3.0f, 2.0f, stream), "grb_luminance_finalize");
		}
		else if (lum)
			cmd.check(grb_luminance(&d3, lum, lerp_lum, -3.0f, 2.0f, stream), "grb_luminance");
		cmd.check(grb_bloom_upsample(&d3, &u2, all_rows(), stream), "grb_bloom_upsample(u2)");
		cmd.check(grb_bloom_upsample(&u2, &u1, all_rows(), stream), "grb_bloom_upsample(u1)");
	}
	// u0 feeds the tonemap's bilinear bloom tap: own band (+ the tonemap halo FXAA needs) at 1/4 res
	if (!tail_fused)
		cmd.check(grb_bloom_upsample_exact(&u1, &u0, u0_rows, stream), "grb_bloom_upsample(u0)"); // the arithmetic the fused tail uses
}

void tonemap_build_render_pass(RenderPass &pass, Vulkan::CommandBuffer &cmd, const RenderTextureResource &hdr_res,
                               const RenderTextureResource &bloom_res, const RenderBufferResource *ubo_res, const HDRDynamicExposureInterface *iface,
                               unsigned)
{
	auto &graph = pass.get_graph();
	GrbImage hdr = graph.get_physical_texture_resource(hdr_res).as_grb();
	GrbImage bloom = graph.get_physical_texture_resource(bloom_res).as_grb();
	const float *lum = ubo_res ? graph.get_physical_buffer_resource(*ubo_res).get<float>() : nullptr;
	auto &out_view = graph.get_physical_texture_resource(*pass.get_color_outputs()[0]);
	GrbImage out = out_view.as_grb();
	float exposure = iface ? iface->get_exposure() : 1.0f; // hdr.cpp:301
	GrbRows rows = graph.is_sharded() ? graph.get_shard_plan().tonemap : GrbRows{ 0, 0 };
	cmd.check(grb_tonemap(&hdr, &bloom, lum, exposure, &out, rows, cmd.get_stream_handle()), "grb_tonemap");
}
} // namespace

void setup_hdr_postprocess_compute(RenderGraph &graph, const FrameParameters &frame, const std::string &input, const std::string &output,
                                   const HDROptions &options, const HDRDynamicExposureInterface *iface)
{
	BufferInfo buffer_info;
	buffer_info.size = 3 * sizeof(float);
	buffer_info.usage = VK_BUFFER_USAGE_STORAGE_BUFFER_BIT | VK_BUFFER_USAGE_UNIFORM_BUFFER_BIT;

	AttachmentInfo downsample_info;
	downsample_info.format = VK_FORMAT_R16G16B16A16_SFLOAT;
	downsample_info.size_x = 0.5f;
	downsample_info.size_y = 0.5f;
	downsample_info.size_class = SizeClass::InputRelative;
	downsample_info.size_relative_name = input;
	downsample_info.aux_usage = VK_IMAGE_USAGE_SAMPLED_BIT;
	auto level = [&](float s) {
		auto info = downsample_info;
		info.size_x = s;
		info.size_y = s;
		return info;
	};

	auto &bloom_pass = graph.add_pass("bloom-compute", RenderGraph::get_default_compute_queue());
	auto res = std::make_shared<BloomResources>();
	res->t = &bloom_pass.add_storage_texture_output("threshold", downsample_info);
	res->d0 = &bloom_pass.add_storage_texture_output("downsample-0", level(0.25f));
	res->u0 = &bloom_pass.add_storage_texture_output("upsample-0", level(0.25f));
	res->d1 = &bloom_pass.add_storage_texture_output("downsample-1", level(0.125f));
	res->u1 = &bloom_pass.add_storage_texture_output("upsample-1", level(0.125f));
	res->d2 = &bloom_pass.add_storage_texture_output("downsample-2", level(0.0625f));
	res->u2 = &bloom_pass.add_storage_texture_output("upsample-2", level(0.0625f));
	res->d3 = &bloom_pass.add_storage_texture_output("downsample-3", level(0.03125f));
	res->lum = nullptr;
	res->lum_grid = nullptr;
	if (options.dynamic_exposure)
	{
		res->lum = &bloom_pass.add_storage_output("average-luminance", buffer_info);
		// scratch for the row-sharded luminance sum: the (d3/2) sample grid (hdr.cpp:78-79), sized from
		// the backbuffer: d3 = ceil(dim / 32)
		BufferInfo grid_info;
		{
			const auto dim = graph.get_backbuffer_dimensions();
			const size_t gx = (size_t(dim.width) + 31) / 32 / 2 + 1, gy = (size_t(dim.height) + 31) / 32 / 2 + 1;
			grid_info.size = std::max<size_t>(gx * gy * sizeof(float), 64 * 1024);
		}
		grid_info.usage = VK_BUFFER_USAGE_STORAGE_BUFFER_BIT;
		res->lum_grid = &bloom_pass.add_storage_output("average-luminance-grid", grid_info);
	}
	res->hdr = &bloom_pass.add_texture_input(input);
	bloom_pass.add_history_input("downsample-3");
	bloom_pass.set_build_render_pass([&graph, &frame, res](Vulkan::CommandBuffer &cmd) { bloom_build_compute(cmd, graph, frame, *res); });

	{
		AttachmentInfo tonemap_info;
		tonemap_info.flags |= ATTACHMENT_INFO_SUPPORTS_PREROTATE_BIT;
		tonemap_info.size_class = SizeClass::InputRelative;
		tonemap_info.size_relative_name = input;
		auto &tonemap = graph.add_pass("tonemap", RenderGraph::get_default_post_graphics_queue());
		tonemap.add_color_output(output, tonemap_info);
		auto &hdr_res = tonemap.add_texture_input(input);
		auto &bloom_res = tonemap.add_texture_input("upsample-0");
		const RenderBufferResource *ubo_res = nullptr;
		if (options.dynamic_exposure)
			ubo_res = &tonemap.add_uniform_input("average-luminance");
		tonemap.set_build_render_pass([&tonemap, &hdr_res, &bloom_res, ubo_res, iface, &graph](Vulkan::CommandBuffer &cmd) {
			// FXAA downstream reads +-9 rows around a band: tonemap that halo too when a consumer declared it
			unsigned halo = graph.find_pass("fxaa") ? 12u : 0u;
			tonemap_build_render_pass(tonemap, cmd, hdr_res, bloom_res, ubo_res, iface, halo);
		});
	}
}

void setup_hdr_postprocess(RenderGraph &graph, const FrameParameters &frame, const std::string &input, const std::string &output,
                           const HDROptions &options, const HDRDynamicExposureInterface *iface)
{
	setup_hdr_postprocess_compute(graph, frame, input, output, options, iface);
}
// ---------------------------------------------------------------------------------------------------- HDR10 / PQ
namespace
{
// Chromaticities (x, y) -> XYZ, Y = 1; then the per-primary scale that makes R+G+B land on the white point
// (renderer/post/hdr.cpp:563-578 through math/transforms' compute_xyz_matrix).  Done in double, as a 4x4 so that the
// host's own Gauss-Jordan inverse serves; rounded to fp32 once at the end.
struct Mat3d
{
	double m[3][3]; // m[col][row]
};

// x = inverse(a) * rhs by Gauss-Jordan elimination with partial pivoting.
void solve3(const Mat3d &m, const double rhs[3], double x[3])
{
	double a[3][4];
	for (int r = 0; r < 3; r++)
	{
		for (int c = 0; c < 3; c++)
			a[r][c] = m.m[c][r];
		a[r][3] = rhs[r];
	}
	for (int k = 0; k < 3; k++)
	{
		int piv = k;
		for (int r = k + 1; r < 3; r++)
			if (std::fabs(a[r][k]) > std::fabs(a[piv][k]))
				piv = r;
		if (piv != k)
			for (int c = 0; c < 4; c++)
				std::swap(a[k][c], a[piv][c]);
		for (int r = 0; r < 3; r++)
		{
			if (r == k)
				continue;
			const double f = a[r][k] / a[k][k];
			for (int c = k; c < 4; c++)
				a[r][c] -= f * a[k][c];
		}
	}
	for (int r = 0; r < 3; r++)
		x[r] = a[r][3] / a[r][r];
}

Mat3d xyz_from_chromaticities(const VkHdrMetadataEXT &md)
{
	const VkXYColorEXT prim[3] = { md.displayPrimaryRed, md.displayPrimaryGreen, md.displayPrimaryBlue };
	Mat3d p;
	for (int c = 0; c < 3; c++)
	{
		const double x = prim[c].x, y = prim[c].y;
		p.m[c][0] = x / y;
		p.m[c][1] = 1.0;
		p.m[c][2] = (1.0 - x - y) / y;
	}
	const double wx = md.whitePoint.x, wy = md.whitePoint.y;
	const double white[3] = { wx / wy, 1.0, (1.0 - wx - wy) / wy };
	double scale[3];
	solve3(p, white, scale);
	for (int c = 0; c < 3; c++)
		for (int r = 0; r < 3; r++)
			p.m[c][r] *= scale[c];
	return p;
}
} // namespace

muglm::mat4 compute_rec709_to_display_primaries(const VkHdrMetadataEXT &metadata)
{
	VkHdrMetadataEXT rec709 = {};
	rec709.displayPrimaryRed = { 0.640f, 0.330f };
	rec709.displayPrimaryGreen = { 0.3f, 0.6f };
	rec709.displayPrimaryBlue = { 0.150f, 0.060f };
	rec709.whitePoint = { 0.3127f, 0.3290f };
	const Mat3d src = xyz_from_chromaticities(rec709), dst = xyz_from_chromaticities(metadata);
	muglm::mat4 out(1.0f); // mat4(mat3): identity elsewhere (hdr.cpp:651)
	for (int col = 0; col < 3; col++)
	{
		double x[3];
		solve3(dst, src.m[col], x); // column of inverse(dst) * src
		for (int r = 0; r < 3; r++)
			out[col][r] = (float)x[r];
	}
	return out;
}

void setup_hdr10_pq_encoding(RenderGraph &graph, const std::string &output, const std::string &hdr_input, const std::string &ui_input,
                             const HDR10PQEncodingConfig &config, const VkHdrMetadataEXT &static_metadata)
{
	struct PQEncoder : RenderPassInterface
	{
		HDR10PQEncodingConfig config = {};
		RenderGraph *graph = nullptr;
		RenderPass *self = nullptr;
		RenderTextureResource *hdr = nullptr;
		RenderTextureResource *ui = nullptr;
		muglm::mat4 primary_conversion;
		float max_light_level = 1000.0f;

		bool get_clear_color(unsigned, VkClearColorValue *) const override { return false; }

		void build_render_pass(Vulkan::CommandBuffer &cmd) override
		{
			GrbImage h = graph->get_physical_texture_resource(*hdr).as_grb();
			GrbImage u = graph->get_physical_texture_resource(*ui).as_grb_unorm();
			GrbImage o = graph->get_physical_texture_resource(*self->get_color_outputs()[0]).as_grb();
			const GrbRows rows = graph->is_sharded() ? graph->get_shard_plan().own : GrbRows{ 0, 0 };
			cmd.check(grb_pq10_encode(&h, &u, primary_conversion.data(), config.hdr_pre_exposure, config.ui_pre_exposure, max_light_level, &o, rows,
			                          cmd.get_stream_handle()),
			          "grb_pq10_encode");
		}
	};

	auto &pq10 = graph.add_pass("pq10", RENDER_GRAPH_QUEUE_GRAPHICS_BIT);
	AttachmentInfo att;
	att.size_class = SizeClass::InputRelative;
	att.size_relative_name = hdr_input;
	att.format = VK_FORMAT_A2B10G10R10_UNORM_PACK32; // the HDR10 swapchain format the reference's default attachment resolves to
	auto pass = std::make_shared<PQEncoder>();
	pass->config = config;
	pass->graph = &graph;
	pass->self = &pq10;
	pass->primary_conversion = compute_rec709_to_display_primaries(static_metadata);
	pass->max_light_level = static_metadata.maxContentLightLevel; // hdr.cpp:652
	pq10.add_color_output(output, att);
	pass->hdr = &pq10.add_texture_input(hdr_input);
	pass->ui = &pq10.add_texture_input(ui_input);
	pq10.set_render_pass_interface(std::move(pass));
}
} // namespace Granite
