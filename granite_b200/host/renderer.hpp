// renderer.hpp -- DeferredLightRenderer::render_light (renderer/renderer.hpp:236,
// renderer/renderer.cpp:1004-1156) and the lighting pass interface that calls it
// (RenderPassSceneRenderer with SCENE_RENDERER_DEFERRED_LIGHTING_BIT,
// renderer/scene_renderer.cpp:483-484), reduced to the hot path: the G-buffer is an input
// (rasterising it is out of scope), the lighting is one C-ABI call.
#pragma once

#include "clusterer.hpp"
#include "render_context.hpp"
#include "render_graph.hpp"

namespace Granite
{
struct GBufferViews
{
	Vulkan::ImageView *albedo = nullptr; // "albedo"  R8G8B8A8_SRGB
	Vulkan::ImageView *normal = nullptr; // "normal"  A2B10G10R10_UNORM
	Vulkan::ImageView *pbr = nullptr;    // "pbr"     R8G8_UNORM
	Vulkan::ImageView *depth = nullptr;  // "depth-transient" D32_SFLOAT
	// "emissive" when HDR-main is a separate image; null when HDR-main aliases it (in-place blend)
	Vulkan::ImageView *emissive = nullptr;
};

class DeferredLightRenderer
{
public:
	// Adds directional + clustered lighting into `hdr` (in place; HDR-main aliases emissive).
	// schedule: optional device buffer of grb_lighting_schedule_bytes(height) bytes kept across frames.
	// stripes: light that stripe set instead of `rows` (grb_deferred_lighting_stripes; row-sharded frames lit in stripes).
	static void render_light(Vulkan::CommandBuffer &cmd, const RenderContext &context, const GBufferViews &gbuffer,
	                         Vulkan::ImageView &hdr, GrbRows rows, void *schedule = nullptr, const GrbStripes *stripes = nullptr);
};

// The "lighting" pass: reads albedo/normal/pbr/depth attachments + the cluster buffers, writes
// HDR-main over emissive (application/scene_viewer_application.cpp:956-975).
class DeferredLightingPass : public RenderPassInterface
{
public:
	DeferredLightingPass(const RenderContext &context_, LightClusterer *clusterer_) : context(context_), clusterer(clusterer_) {}
	void setup_dependencies(RenderPass &self, RenderGraph &graph) override;
	void build_render_pass(Vulkan::CommandBuffer &cmd) override;
	void set_resources(RenderGraph &graph_, RenderTextureResource &albedo, RenderTextureResource &normal, RenderTextureResource &pbr,
	                   RenderTextureResource &depth, RenderTextureResource &hdr, RenderTextureResource *emissive = nullptr);

private:
	const RenderContext &context;
	LightClusterer *clusterer;
	RenderGraph *graph = nullptr;
	RenderTextureResource *res_albedo = nullptr, *res_normal = nullptr, *res_pbr = nullptr, *res_depth = nullptr, *res_hdr = nullptr;
	RenderTextureResource *res_emissive = nullptr;
	RenderBufferResource *res_schedule = nullptr;
	unsigned halo_rows = 0;

public:
	// extra rows around a row shard that downstream passes (bloom threshold, FXAA) read
	void set_shard_halo(unsigned rows) { halo_rows = rows; }
	void set_schedule(RenderBufferResource &schedule) { res_schedule = &schedule; }
	// Row-sharded frames lit in stripes: the pass lights `stripes` instead of its lighting rows, then calls `push` on
	// the same stream with HDR-main (the rows the other ranks read go to them: scene_viewer.cpp).
	void set_stripes(GrbStripes stripes_, std::function<void(Vulkan::CommandBuffer &, Vulkan::ImageView &)> push_)
	{
		stripes = stripes_;
		push = std::move(push_);
	}

private:
	GrbStripes stripes = {};
	std::function<void(Vulkan::CommandBuffer &, Vulkan::ImageView &)> push;
};
} // namespace Granite
