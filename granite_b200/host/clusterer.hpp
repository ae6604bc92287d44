// clusterer.hpp -- LightClusterer for the bindless path (renderer/lights/clusterer.hpp:38-107):
// gathers the visible positional lights front-to-back, fills the parameter/transform blocks,
// declares the "clustering-bindless" pass and, in its callback, uploads the per-frame light
// data and launches the four clusterer kernels through the C ABI.  Shadow-map rendering,
// decals, volumetrics of the reference's class are outside the hot path (SURVEY.md §2).
#pragma once

#include <functional>
#include <memory>
#include <vector>

#include "lights.hpp"
#include "render_graph.hpp"

namespace Granite
{
// math/render_parameters.hpp:146-148
enum
{
	ClustererMaxLightsBindless = 4096
};

struct PositionalLightInfo
{
	PositionalLight *light;
	mat_affine transform; // node world transform
};
using PositionalLightList = std::vector<PositionalLightInfo>;

class LightClusterer
{
public:
	LightClusterer();
	~LightClusterer();

	void set_resolution(unsigned x, unsigned y, unsigned z);
	void set_enable_clustering(bool enable) { enable_clustering = enable; }
	// Declare the clustering pass on RENDER_GRAPH_QUEUE_ASYNC_COMPUTE_BIT (second CUDA stream).
	void set_async_compute(bool enable) { async_compute = enable; }
	// Row-sharded frames: only the cluster tiles under pixel rows [y0, y1) of a frame `height` rows tall are consumed
	// by this rank's lighting pass, so only those tile rows are binned (one tile row of margin either side).
	// y1 <= y0: every row (default).
	void set_lit_pixel_rows(int y0, int y1, int height)
	{
		lit_y0 = y0;
		lit_y1 = y1;
		lit_height = height;
	}
	// Row-sharded frames lit in stripes: the tile-row ranges under this rank's stripes (StripePlan::tile_rows), binned
	// one range at a time; they replace the lit pixel rows above.  Empty: off (default).
	void set_lit_tile_ranges(std::vector<GrbRows> ranges) { lit_tile_ranges = std::move(ranges); }
	// Shadowed positional lights (clusterer.cpp:78-81,173-176): the lighting pass multiplies each light by the PCF
	// comparison sample of its shadow map (PositionalLight::set_shadow_map).  RENDERING the maps is the caller's
	// (clusterer.cpp:206-330 is rasterisation, outside the path); for scene lights the clusterer computes the per-light
	// shadow transforms (clusterer.cpp:467-474 spot, :518-521 point) and uploads them with the map pointers; device
	// lights bring their own (DeviceLightSource::shadows).
	void set_enable_shadows(bool enable) { enable_shadows = enable; }
	bool get_enable_shadows() const { return enable_shadows; }
	void set_shadow_resolution(unsigned res) { shadow_resolution = res; }
	unsigned get_shadow_resolution() const { return shadow_resolution; }
	// config "PCFKernelWide" (scene_viewer_application.cpp:208-217 -> Renderer::SHADOW_PCF_KERNEL_WIDE_BIT)
	void set_shadow_pcf_kernel_wide(bool enable) { shadow_pcf_wide = enable; }
	// ClustererBindlessTransforms::shadow[index] of a spot light (xy_range = SpotLight::get_xy_range) / a point light
	static mat4 spot_shadow_transform(const PositionalFragmentInfo &light, float xy_range);
	static mat4 point_shadow_transform(const PositionalFragmentInfo &light);
	// The C-ABI view of the uploaded shadow data (null members while shadows are disabled).
	GrbLightShadows get_light_shadows() const;
	const std::vector<mat4> &get_shadow_transforms() const { return shadow_transforms; }
	const std::vector<const void *> &get_shadow_maps() const { return shadow_maps; }
	// Volumetric decals (clusterer.cpp:148-156, 1348-1461): binned over the same tile grid and Z slices as the lights, into
	// "cluster-bitmask-decal" / "cluster-range-decal".  The scene's decals are their world transforms (unit cubes in decal
	// space; replaces Scene::gather_visible_volumetric_decals): culled against the frustum, sorted by view depth of their
	// centre, at most MaxDecalsBindless.  Sampling the decal textures is the material pass's job, outside the path.
	enum
	{
		MaxDecalsBindless = 4096
	};
	void set_enable_volumetric_decals(bool enable) { enable_volumetric_decals = enable; }
	bool clusterer_has_volumetric_decals() const { return enable_volumetric_decals; }
	void set_scene_decals(const std::vector<mat_affine> *world_transforms) { scene_decals = world_transforms; }
	const Vulkan::Buffer *get_cluster_bitmask_decal_buffer() const { return bitmask_decal_buffer; }
	const Vulkan::Buffer *get_cluster_range_decal_buffer() const { return range_decal_buffer; }
	unsigned get_active_decal_count() const { return (unsigned)decal_mvps.size(); }
	// CPU copies of what is uploaded (parity tests): view_projection * world per visible decal, and the Z-slice ranges
	const std::vector<mat4> &get_decal_mvps() const { return decal_mvps; }
	const std::vector<uvec2> &get_decal_z_ranges() const { return decal_index_range; }
	static vec2 decal_z_range(const RenderContext &context, const mat_affine &transform);
	void set_max_spot_lights(unsigned) {}
	void set_max_point_lights(unsigned) {}

	// The scene's positional lights (replaces the ECS gather in renderer/threaded_scene.cpp:112-153).
	void set_scene_lights(const PositionalLightList *lights) { scene_lights = lights; }
	// Lights that live in device memory: while a source is set the scene lights are ignored, refresh() fills only the
	// parameters (num_lights = min(count, ClustererMaxLightsBindless) slots) and the clustering pass culls, sorts and
	// packs the list on the device (grb_light_prep) before the four kernels, K3 in its counted form.  The kept count
	// stays on the device at `count`.  `ready` (a cudaEvent_t or null) is waited on before the first read of the
	// arrays and `consumed` recorded after the last.  With shadows enabled the caller also gives each input light's
	// shadow transform and map (`shadows`, read under the same events): the prep (grb_light_prep_shadowed) moves them into
	// cluster order, into the tables get_light_shadows() points at.  The transforms are the caller's, never computed here.
	// `input_count` (device, or null = all list.count entries are lights) makes list.count a capacity: the prep
	// (grb_light_prep[_shadowed]_counted) reads the live length under the same events; refresh() still sizes the frame
	// from the capacity.
	// With `by_id` the maps come by map id instead (grb_light_prep_shadow_ids): `shadow_ids` holds each input light's
	// transform and id, and `map_table` (device, `map_table_size` entries) turns an id into this rank's map.
	// Row-sharded frames whose list comes from one rank (scene_viewer.cpp, grbh_viewer_set_light_source_rank):
	// `exchange` runs on the pass's stream after `ready` and may replace the list, count and shadow ids the prep reads
	// with this frame's received copy; `after_prep` runs right behind the prep, before `consumed` and the cluster kernels.
	struct DeviceLightSource
	{
		GrbLightList list = {};
		GrbLightShadowList shadows = {};
		bool by_id = false;
		GrbLightShadowIdList shadow_ids = {};
		const void *const *map_table = nullptr;
		int32_t map_table_size = 0;
		const int32_t *input_count = nullptr;
		std::function<void(Vulkan::CommandBuffer &, GrbLightList &, const int32_t *&, GrbLightShadowIdList &)> exchange;
		std::function<void(Vulkan::CommandBuffer &)> after_prep;
		void *ready = nullptr, *consumed = nullptr;
		void *scratch = nullptr; // grb_light_prep_scratch_bytes(list.count) or more
		size_t scratch_bytes = 0;
		int32_t *count = nullptr; // device
	};
	void set_device_lights(const DeviceLightSource *source) { device_lights = source; }
	bool has_device_lights() const { return device_lights != nullptr; }
	// the reference always culls the light list against the camera frustum (scene.cpp:333-358)
	void set_enable_frustum_culling(bool enable) { frustum_culling = enable; }

	// RenderPassCreator surface
	void add_render_passes(RenderGraph &graph);
	void setup_render_pass_dependencies(RenderGraph &graph, RenderPass &target);
	void setup_render_pass_resources(RenderGraph &graph);
	void set_base_render_context(const RenderContext *context_) { context = context_; }

	// PerFrameRefreshable: sort + scan lights, fill parameters (clusterer.cpp:1133-1176, 781-889).
	void refresh(const RenderContext &context);

	const GrbClusterParameters &get_cluster_parameters_bindless() const { return parameters; }
	const Vulkan::Buffer *get_cluster_transform_buffer() const { return transforms_buffer; }
	const Vulkan::Buffer *get_cluster_bitmask_buffer() const { return bitmask_buffer; }
	const Vulkan::Buffer *get_cluster_range_buffer() const { return range_buffer; }
	// The C-ABI view of the graph-owned cluster buffers (valid after setup_render_pass_resources).
	GrbClusterBuffers get_cluster_buffers() const;
	unsigned get_active_light_count() const { return (unsigned)parameters.num_lights; }

	// CPU copies of what is uploaded each frame (exposed for the parity tests).
	const std::vector<PositionalFragmentInfo> &get_light_records() const { return lights; }
	const std::vector<mat_affine> &get_model_transforms() const { return model; }
	const std::vector<uint32_t> &get_type_mask() const { return type_mask; }
	const std::vector<uvec2> &get_z_ranges() const { return volume_index_range; }

private:
	const RenderContext *context = nullptr;
	const PositionalLightList *scene_lights = nullptr;
	const DeviceLightSource *device_lights = nullptr;
	GrbLightPrepView device_view = {};
	bool frustum_culling = true;
	std::vector<uint8_t> visible;
	unsigned resolution_x = 64, resolution_y = 32, resolution_z = 16;
	bool enable_clustering = true;
	bool async_compute = false;
	int lit_y0 = 0, lit_y1 = 0, lit_height = 0;
	std::vector<GrbRows> lit_tile_ranges;

	GrbClusterParameters parameters = {};
	std::vector<PositionalFragmentInfo> lights;
	std::vector<mat_affine> model;
	std::vector<uint32_t> type_mask;
	std::vector<uvec2> volume_index_range;
	bool enable_shadows = false;
	unsigned shadow_resolution = 512;
	bool shadow_pcf_wide = false;
	std::vector<mat4> shadow_transforms;
	std::vector<const void *> shadow_maps;
	bool enable_volumetric_decals = false;
	const std::vector<mat_affine> *scene_decals = nullptr;
	std::vector<mat4> decal_mvps;
	std::vector<uvec2> decal_index_range;
	RenderBufferResource *res_bitmask_decal = nullptr, *res_range_decal = nullptr, *res_decal_scratch = nullptr;
	const Vulkan::Buffer *bitmask_decal_buffer = nullptr, *range_decal_buffer = nullptr, *decal_scratch_buffer = nullptr;
	void refresh_decals(const RenderContext &ctx);
	void build_decal_clusters_gpu(Vulkan::CommandBuffer &cmd);
	std::vector<unsigned> sort_order;
	std::vector<float> sort_keys;
	// pinned staging copy of {lights, model, type_mask, z ranges} for the async upload
	void *staging = nullptr;
	size_t staging_size = 0;
	void *staging_events[2] = { nullptr, nullptr };
	bool staging_event_pending[2] = { false, false };
	unsigned staging_slot = 0;

	RenderBufferResource *res_bitmask = nullptr, *res_range = nullptr, *res_transforms = nullptr;
	RenderBufferResource *res_cull = nullptr, *res_spots = nullptr;
	const Vulkan::Buffer *bitmask_buffer = nullptr, *range_buffer = nullptr, *transforms_buffer = nullptr;
	const Vulkan::Buffer *cull_buffer = nullptr, *spot_buffer = nullptr;

	float get_z_slice_extent(const RenderContext &ctx) const;
	uvec2 compute_uint_range(vec2 range) const;
	void refresh_bindless_prepare(const RenderContext &ctx);
	void build_cluster_bindless_gpu(Vulkan::CommandBuffer &cmd);
	void launch_cluster_kernels(Vulkan::CommandBuffer &cmd, const int32_t *device_count, int32_t num_ranges);
	void add_render_passes_bindless(RenderGraph &graph);
	size_t transforms_offset_model() const;
	size_t transforms_offset_type_mask() const;
	size_t transforms_size() const;
};
} // namespace Granite
