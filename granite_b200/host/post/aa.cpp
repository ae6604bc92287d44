// aa.cpp -- dispatch of PostAAType to the pass builders (renderer/post/aa.cpp:176-290).
#include "aa.hpp"

#include <stdexcept>

#include "fxaa.hpp"
#include "smaa.hpp"

namespace Granite
{
bool setup_before_post_chain_antialiasing(PostAAType type, RenderGraph &graph, TemporalJitter &jitter, float scaling_factor, const std::string &input,
                                          const std::string &input_depth, const std::string &input_mv, const std::string &output)
{
	switch (type)
	{
	case PostAAType::TAA_Low:
		setup_taa_resolve(graph, jitter, scaling_factor, input, input_depth, input_mv, output, TAAQuality::Low);
		return true;
	case PostAAType::TAA_Medium:
		setup_taa_resolve(graph, jitter, scaling_factor, input, input_depth, input_mv, output, TAAQuality::Medium);
		return true;
	case PostAAType::TAA_High:
		setup_taa_resolve(graph, jitter, scaling_factor, input, input_depth, input_mv, output, TAAQuality::High);
		return true;
	default:
		jitter.init(TemporalJitter::Type::None, vec2(0.0f));
		return false;
	}
}

bool setup_after_post_chain_antialiasing(PostAAType type, RenderGraph &graph, TemporalJitter &jitter, float scaling_factor, const std::string &input,
                                         const std::string &input_depth, const std::string &output)
{
	switch (type)
	{
	case PostAAType::FXAA:
		setup_fxaa_postprocess(graph, input, output);
		return true;
	case PostAAType::SMAA_Low:
		setup_smaa_postprocess(graph, jitter, scaling_factor, input, input_depth, output, SMAAPreset::Low);
		return true;
	case PostAAType::SMAA_Medium:
		setup_smaa_postprocess(graph, jitter, scaling_factor, input, input_depth, output, SMAAPreset::Medium);
		return true;
	case PostAAType::SMAA_High:
		setup_smaa_postprocess(graph, jitter, scaling_factor, input, input_depth, output, SMAAPreset::High);
		return true;
	case PostAAType::SMAA_Ultra:
		setup_smaa_postprocess(graph, jitter, scaling_factor, input, input_depth, output, SMAAPreset::Ultra);
		return true;
	case PostAAType::None:
	case PostAAType::TAA_Low:
	case PostAAType::TAA_Medium:
	case PostAAType::TAA_High:
		return false;
	default:
		throw std::logic_error("PostAAType not supported by this executor (FXAA_2Phase and SMAA T2X are not built).");
	}
}

// renderer/post/aa.cpp:75-174.  The constant blocks (FsrEasuCon, FsrRcasCon: aa.cpp:33-73) are evaluated inside the two
// C-ABI calls from the image sizes and the sharpness, as the reference evaluates them inside its callbacks.
bool setup_after_post_chain_upscaling(RenderGraph &graph, const std::string &input, const std::string &output, bool use_sharpen)
{
	auto &upscale = graph.add_pass(output + "-scale", RenderGraph::get_default_post_graphics_queue());
	AttachmentInfo upscale_info; // swapchain-relative, scale 1: the display size
	upscale_info.flags |= !use_sharpen ? ATTACHMENT_INFO_SUPPORTS_PREROTATE_BIT : 0;
	upscale_info.format = VK_FORMAT_R8G8B8A8_UNORM;
	upscale_info.flags |= use_sharpen ? ATTACHMENT_INFO_UNORM_SRGB_ALIAS_BIT : 0;
	auto &upscale_out = upscale.add_color_output(use_sharpen ? (output + "-scale") : output, upscale_info);
	auto &tex = upscale.add_texture_input(input);
	graph.get_texture_resource(input).get_attachment_info().flags |= ATTACHMENT_INFO_UNORM_SRGB_ALIAS_BIT;
	upscale.set_build_render_pass([&graph, &tex, &upscale_out](Vulkan::CommandBuffer &cmd) {
		// cmd.set_unorm_texture(0, 0, view) + NearestClamp; TARGET_SRGB follows the output's format
		GrbImage in = graph.get_physical_texture_resource(tex).as_grb_unorm();
		GrbImage out = graph.get_physical_texture_resource(upscale_out).as_grb();
		// row-sharded: the band, +-1 row for RCAS (shard_plan.hpp); the input holds the render rows those read
		const GrbRows rows = graph.is_sharded() && graph.get_shard_count() > 1 ? graph.get_shard_plan().easu : GrbRows{ 0, 0 };
		cmd.check(grb_fsr_upscale(&in, &out, rows, cmd.get_stream_handle()), "grb_fsr_upscale");
	});

	if (use_sharpen)
	{
		AttachmentInfo sharpen_info;
		sharpen_info.flags |= ATTACHMENT_INFO_SUPPORTS_PREROTATE_BIT;
		auto &sharpen = graph.add_pass(output + "-sharpen", RenderGraph::get_default_post_graphics_queue());
		auto &sharpen_out = sharpen.add_color_output(output, sharpen_info);
		auto &upscaled = sharpen.add_texture_input(output + "-scale");
		sharpen.set_build_render_pass([&graph, &upscaled, &sharpen_out](Vulkan::CommandBuffer &cmd) {
			// sRGB target: the input is bound through an sRGB view (set_srgb_texture), UNORM otherwise; the kernel
			// picks the view from the OUTPUT's format, so the input descriptor only carries the memory
			GrbImage in = graph.get_physical_texture_resource(upscaled).as_grb();
			GrbImage out = graph.get_physical_texture_resource(sharpen_out).as_grb();
			const GrbRows rows = graph.is_sharded() && graph.get_shard_count() > 1 ? graph.get_shard_plan().own : GrbRows{ 0, 0 };
			cmd.check(grb_fsr_sharpen(&in, &out, 0.5f, rows, cmd.get_stream_handle()), "grb_fsr_sharpen");
		});
	}
	return true;
}
} // namespace Granite
