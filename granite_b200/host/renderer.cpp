#include "renderer.hpp"

#include <cstring>

namespace Granite
{
void DeferredLightRenderer::render_light(Vulkan::CommandBuffer &cmd, const RenderContext &context, const GBufferViews &gb, Vulkan::ImageView &hdr,
                                         GrbRows rows, void *schedule, const GrbStripes *stripes)
{
	auto *light = context.get_lighting_parameters();
	if (!light || !gb.albedo || !gb.normal || !gb.pbr || !gb.depth)
	{
		Vulkan::log_error("render_light: lighting parameters or G-buffer attachment missing.\n");
		return;
	}
	const auto &rp = context.get_render_parameters();

	GrbGBuffer g = {};
	g.albedo = gb.albedo->as_grb();
	g.normal = gb.normal->as_grb();
	g.pbr = gb.pbr->as_grb();
	g.depth = gb.depth->as_grb();
	if (gb.emissive)
		g.emissive = gb.emissive->as_grb();
	// DirectionalLightPush (renderer.cpp:1073-1103)
	for (int i = 0; i < 3; i++)
	{
		g.directional_color[i] = light->directional.color[i];
		g.directional_direction[i] = light->directional.direction[i];
	}

	GrbCamera cam = {};
	std::memcpy(cam.view, rp.view.data(), 64);
	std::memcpy(cam.view_projection, rp.view_projection.data(), 64);
	std::memcpy(cam.inv_view_projection, rp.inv_view_projection.data(), 64);
	for (int i = 0; i < 3; i++)
	{
		cam.camera_position[i] = rp.camera_position[i];
		cam.camera_front[i] = rp.camera_front[i];
	}
	cam.z_near = rp.z_near;
	cam.z_far = rp.z_far;

	GrbClusterParameters params = {};
	GrbClusterBuffers buffers = {};
	if (light->cluster && light->cluster->get_cluster_bitmask_buffer())
	{
		params = light->cluster->get_cluster_parameters_bindless();
		buffers = light->cluster->get_cluster_buffers();
	}
	else
	{
		Vulkan::log_error("render_light: no light cluster bound; the clustered term needs the cluster-range buffer.\n");
		return;
	}
	GrbImage hdr_img = hdr.as_grb();
	// POSITIONAL_LIGHTS_SHADOW (renderer.cpp:1124-1131): the clusterer holds the shadow transforms and map pointers
	const GrbLightShadows shadows = light->cluster->get_light_shadows();
	if (stripes)
		cmd.check(grb_deferred_lighting_stripes(&g, &cam, &params, &buffers, shadows.maps ? &shadows : nullptr, &hdr_img, *stripes, schedule,
		                                        cmd.get_stream_handle()),
		          "grb_deferred_lighting_stripes");
	else if (shadows.maps)
		cmd.check(grb_deferred_lighting_shadowed(&g, &cam, &params, &buffers, &shadows, &hdr_img, rows, cmd.get_stream_handle()), "grb_deferred_lighting_shadowed");
	else
		cmd.check(grb_deferred_lighting_scheduled(&g, &cam, &params, &buffers, &hdr_img, rows, schedule, cmd.get_stream_handle()), "grb_deferred_lighting");
}

void DeferredLightingPass::setup_dependencies(RenderPass &self, RenderGraph &graph_)
{
	// scene.add_render_pass_dependencies(lighting, LIGHTING_BIT) -> clusterer adds its storage inputs
	if (clusterer)
		clusterer->setup_render_pass_dependencies(graph_, self);
	// The persistent kernel takes every SM it is given: let the previous frame's full-machine bloom kernel finish
	// first (host/post/hdr.cpp signals the mark); the latency-bound rest of that chain then runs beside this pass.
	self.add_wait_mark("bloom-head");
}

void DeferredLightingPass::set_resources(RenderGraph &graph_, RenderTextureResource &albedo, RenderTextureResource &normal, RenderTextureResource &pbr,
                                         RenderTextureResource &depth, RenderTextureResource &hdr, RenderTextureResource *emissive)
{
	res_emissive = emissive;
	graph = &graph_;
	res_albedo = &albedo;
	res_normal = &normal;
	res_pbr = &pbr;
	res_depth = &depth;
	res_hdr = &hdr;
}

void DeferredLightingPass::build_render_pass(Vulkan::CommandBuffer &cmd)
{
	GBufferViews gb;
	gb.albedo = &graph->get_physical_texture_resource(*res_albedo);
	gb.normal = &graph->get_physical_texture_resource(*res_normal);
	gb.pbr = &graph->get_physical_texture_resource(*res_pbr);
	gb.depth = &graph->get_physical_texture_resource(*res_depth);
	if (res_emissive)
		gb.emissive = &graph->get_physical_texture_resource(*res_emissive);
	auto &hdr = graph->get_physical_texture_resource(*res_hdr);
	void *schedule = res_schedule ? graph->get_physical_buffer_resource(*res_schedule).get_device_pointer() : nullptr;
	if (push)
	{
		DeferredLightRenderer::render_light(cmd, context, gb, hdr, GrbRows{ 0, 0 }, schedule, &stripes);
		push(cmd, hdr);
		return;
	}
	DeferredLightRenderer::render_light(cmd, context, gb, hdr, graph->is_sharded() ? graph->get_shard_plan().lighting : GrbRows{ 0, 0 }, schedule);
}
} // namespace Granite
