// smaa.cpp -- "smaa-edge" / "smaa-weights" / "smaa-blend" pass builders (renderer/post/smaa.cpp:32-209), the lookup
// textures they sample and the .gtx reader for them.
//
// Row-sharded frames (shard_plan.hpp derives the rows): a rank detects the edges of its own rows, and its weight pass
// needs a window of up to 2 * max_search_steps + 6 rows around its band, mostly other ranks' rows.  The edge kernel
// stores each row straight into the edge image of every rank whose window holds it (NVLink peer memory, the SMAA
// channel of RenderGraphCollectives) and raises a flag; the weight pass waits for every rank's flag and reads that
// copy.  Without peer memory: the plain edge kernel, then the ranks' edge bands are all-gathered with NCCL.
#include "smaa.hpp"

#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>

namespace Granite
{
namespace
{
struct Lookup
{
	Vulkan::ImageHandle area, search;
};
std::mutex g_lookup_lock;
std::map<Vulkan::Device *, Lookup> g_lookup;

constexpr unsigned kAreaW = 160, kAreaH = 560, kSearchW = 64, kSearchH = 16;
} // namespace

bool set_smaa_lookup_textures(Vulkan::Device &device, const uint8_t *area_rg8, const uint8_t *search_r8)
{
	if (!area_rg8 || !search_r8)
		return false;
	Lookup l;
	Vulkan::ImageCreateInfo info;
	info.width = kAreaW;
	info.height = kAreaH;
	info.format = VK_FORMAT_R8G8_UNORM;
	l.area = device.create_image(info);
	info.width = kSearchW;
	info.height = kSearchH;
	info.format = VK_FORMAT_R8_UNORM;
	l.search = device.create_image(info);
	// once per device, before the first frame: plain synchronous copies.  create_image zero-fills on the device's
	// stream, which the legacy-stream copies below do not wait for: finish the fill first, or it can land after the
	// upload and leave zero lookup textures (no SMAA weights at all).
	device.wait_idle();
	if (!Vulkan::cuda_ok(cudaMemcpy(l.area->get_device_pointer(), area_rg8, (size_t)kAreaW * kAreaH * 2, cudaMemcpyHostToDevice), "SMAA area texture upload") ||
	    !Vulkan::cuda_ok(cudaMemcpy(l.search->get_device_pointer(), search_r8, (size_t)kSearchW * kSearchH, cudaMemcpyHostToDevice), "SMAA search texture upload"))
		return false;
	std::lock_guard<std::mutex> hold(g_lookup_lock);
	g_lookup[&device] = std::move(l);
	return true;
}

bool get_smaa_lookup_textures(Vulkan::Device &device, GrbImage *area, GrbImage *search)
{
	std::lock_guard<std::mutex> hold(g_lookup_lock);
	auto itr = g_lookup.find(&device);
	if (itr == g_lookup.end())
		return false;
	*area = Vulkan::ImageView(itr->second.area).as_grb();
	*search = Vulkan::ImageView(itr->second.search).as_grb();
	return true;
}

void release_smaa_lookup_textures(Vulkan::Device &device)
{
	std::lock_guard<std::mutex> hold(g_lookup_lock);
	g_lookup.erase(&device);
}

bool parse_gtx(const uint8_t *bytes, size_t size, GtxImage &out, std::string &error)
{
	static const char magic[16] = "GRANITE TEXFMT1";
	if (!bytes || size < 64 || std::memcmp(bytes, magic, 16) != 0)
	{
		error = "not a GRANITE TEXFMT1 container";
		return false;
	}
	uint32_t h[8];
	uint64_t payload = 0;
	std::memcpy(h, bytes + 16, sizeof(h));
	std::memcpy(&payload, bytes + 48, 8);
	const uint32_t type = h[0], format = h[1], width = h[2], height = h[3], depth = h[4], layers = h[5], levels = h[6];
	if (type != 1 /* VK_IMAGE_TYPE_2D */ || depth != 1 || layers != 1 || levels != 1 || width == 0 || height == 0)
	{
		error = "only single-level, single-layer 2-D images are read";
		return false;
	}
	const unsigned texel = format_texel_size((VkFormat)format);
	if (!texel)
	{
		error = "texel format not handled by this executor";
		return false;
	}
	const size_t need = (size_t)width * height * texel;
	if (payload < need || size < 64 + need)
	{
		error = "payload shorter than width x height texels";
		return false;
	}
	out.format = (VkFormat)format;
	out.width = width;
	out.height = height;
	out.texels.assign(bytes + 64, bytes + 64 + need);
	return true;
}

bool load_gtx(const std::string &path, GtxImage &out, std::string &error)
{
	std::FILE *f = std::fopen(path.c_str(), "rb");
	if (!f)
	{
		error = "cannot open " + path;
		return false;
	}
	std::vector<uint8_t> bytes;
	uint8_t chunk[65536];
	size_t n;
	while ((n = std::fread(chunk, 1, sizeof(chunk), f)) > 0)
		bytes.insert(bytes.end(), chunk, chunk + n);
	std::fclose(f);
	if (!parse_gtx(bytes.data(), bytes.size(), out, error))
	{
		error = path + ": " + error;
		return false;
	}
	return true;
}

bool load_smaa_lookup_textures(Vulkan::Device &device, const std::string &directory, std::string &error)
{
	GtxImage area, search;
	if (!load_gtx(directory + "/area.gtx", area, error) || !load_gtx(directory + "/search.gtx", search, error))
		return false;
	if (area.format != VK_FORMAT_R8G8_UNORM || area.width != kAreaW || area.height != kAreaH || search.format != VK_FORMAT_R8_UNORM || search.width != kSearchW ||
	    search.height != kSearchH)
	{
		error = "area.gtx must be 160x560 R8G8_UNORM and search.gtx 64x16 R8_UNORM";
		return false;
	}
	if (!set_smaa_lookup_textures(device, area.texels.data(), search.texels.data()))
	{
		error = "upload of the SMAA lookup textures failed";
		return false;
	}
	return true;
}

void setup_smaa_postprocess(RenderGraph &graph, TemporalJitter &jitter, float, const std::string &input, const std::string &, const std::string &output,
                            SMAAPreset preset)
{
	if (preset == SMAAPreset::Ultra_T2X)
		throw std::logic_error("SMAA T2X (two jittered frames + smaa-t2x-resolve) is not built by this executor.");
	const int quality = preset == SMAAPreset::Low ? 0 : (preset == SMAAPreset::Medium ? 1 : (preset == SMAAPreset::High ? 2 : 3));
	jitter.init(TemporalJitter::Type::None, vec2(1.0f)); // smaa.cpp:66-67

	// the input is sampled through a UNORM view of its sRGB storage (smaa.cpp:70, 124, 178)
	graph.get_texture_resource(input).get_attachment_info().flags |= ATTACHMENT_INFO_UNORM_SRGB_ALIAS_BIT;

	AttachmentInfo edge_info;
	edge_info.size_class = SizeClass::InputRelative;
	edge_info.size_relative_name = input;
	edge_info.format = VK_FORMAT_R8G8_UNORM;
	AttachmentInfo weight_info = edge_info;
	weight_info.format = VK_FORMAT_R8G8B8A8_UNORM;
	AttachmentInfo final_info;
	final_info.size_class = SizeClass::InputRelative;
	final_info.size_relative_name = input;

	auto &smaa_edge = graph.add_pass("smaa-edge", RenderGraph::get_default_post_graphics_queue());
	auto &smaa_weight = graph.add_pass("smaa-weights", RenderGraph::get_default_post_graphics_queue());
	auto &smaa_blend = graph.add_pass("smaa-blend", RenderGraph::get_default_post_graphics_queue());

	// The reference also attaches a D16 "smaa-mask" to the first two passes (smaa.cpp:101-118, 148-149): both draw at
	// depth 0, which is the clear value, so the EQUAL test of the second pass keeps every pixel -- nothing to carry over.
	auto &edge_out = smaa_edge.add_color_output("smaa-edge", edge_info);
	auto &edge_input = smaa_edge.add_texture_input(input);
	auto &weight_out = smaa_weight.add_color_output("smaa-weights", weight_info);
	auto &weight_input = smaa_weight.add_texture_input("smaa-edge");
	auto &blend_out = smaa_blend.add_color_output(output, final_info);
	auto &blend_input = smaa_blend.add_texture_input(input);
	auto &blend_weights = smaa_blend.add_texture_input("smaa-weights");

	// this frame's slot of the edge exchange, from the edge pass to the weight pass (both on the post-graphics stream)
	struct EdgeExchange
	{
		bool peer_stores = false;
		RenderGraphCollectives::PeerSlot slot;
	};
	auto exchange = std::make_shared<EdgeExchange>();
	smaa_edge.set_build_render_pass([&graph, &edge_out, &edge_input, quality, exchange](Vulkan::CommandBuffer &cmd) {
		GrbImage color = graph.get_physical_texture_resource(edge_input).as_grb_unorm();
		auto &edge_view = graph.get_physical_texture_resource(edge_out);
		GrbImage edges = edge_view.as_grb();
		void *stream = cmd.get_stream_handle();
		const bool sharded = graph.is_sharded() && graph.get_shard_count() > 1;
		exchange->peer_stores = sharded && graph.get_collectives()->peer_exchange_begin_frame(RenderGraphCollectives::PeerChannel::SmaaEdges,
		                                                                                      (size_t)edges.row_pitch * (size_t)edges.height, exchange->slot);
		if (!sharded)
		{
			cmd.check(grb_smaa_edge_detection(&color, quality, &edges, GrbRows{ 0, 0 }, stream), "grb_smaa_edge_detection");
			return;
		}
		const std::vector<GrbRows> bands = graph.get_shard_plan_rows(&ShardPlan::smaa_edges);
		const unsigned self = graph.get_shard_rank();
		if (exchange->peer_stores)
		{
			const auto &slot = exchange->slot;
			const std::vector<GrbRows> windows = graph.get_shard_plan_rows(&ShardPlan::smaa_edge_window);
			cmd.check(grb_smaa_edge_detection_to_peers(&color, quality, &edges, slot.images, slot.flags, windows.data(), (int32_t)slot.count, (int32_t)self,
			                                           slot.epoch, slot.counter, bands[self], stream),
			          "grb_smaa_edge_detection_to_peers");
			return;
		}
		cmd.check(grb_smaa_edge_detection(&color, quality, &edges, bands[self], stream), "grb_smaa_edge_detection");
		graph.get_collectives()->all_gather_rows(cmd, edge_view, bands);
	});
	smaa_weight.set_build_render_pass([&graph, &weight_out, &weight_input, quality, exchange](Vulkan::CommandBuffer &cmd) {
		GrbImage edges = graph.get_physical_texture_resource(weight_input).as_grb();
		GrbImage weights = graph.get_physical_texture_resource(weight_out).as_grb();
		GrbImage area, search;
		if (!get_smaa_lookup_textures(cmd.get_device(), &area, &search))
		{
			Vulkan::log_error("smaa-weights: no lookup textures on this device (set_smaa_lookup_textures / load_smaa_lookup_textures).\n");
			return;
		}
		void *stream = cmd.get_stream_handle();
		const bool sharded = graph.is_sharded() && graph.get_shard_count() > 1;
		if (sharded && exchange->peer_stores)
		{
			const auto &slot = exchange->slot;
			const unsigned self = graph.get_shard_rank();
			cmd.check(grb_peer_wait(slot.flags[self], (int32_t)slot.count, slot.epoch, stream), "grb_peer_wait");
			edges.data = slot.images[self]; // the exchanged copy
		}
		const GrbRows rows = sharded ? graph.get_shard_plan().smaa_weights : GrbRows{ 0, 0 };
		cmd.check(grb_smaa_blend_weights(&edges, &area, &search, quality, &weights, rows, stream), "grb_smaa_blend_weights");
	});
	smaa_blend.set_build_render_pass([&graph, &blend_out, &blend_input, &blend_weights](Vulkan::CommandBuffer &cmd) {
		GrbImage color = graph.get_physical_texture_resource(blend_input).as_grb_unorm();
		GrbImage weights = graph.get_physical_texture_resource(blend_weights).as_grb();
		GrbImage out = graph.get_physical_texture_resource(blend_out).as_grb(); // SMAA_TARGET_SRGB follows the output format (smaa.cpp:193-194)
		const GrbRows rows = graph.is_sharded() && graph.get_shard_count() > 1 ? graph.get_shard_plan().smaa_blend : GrbRows{ 0, 0 };
		cmd.check(grb_smaa_neighborhood_blend(&color, &weights, &out, rows, cmd.get_stream_handle()), "grb_smaa_neighborhood_blend");
	});
}
} // namespace Granite
