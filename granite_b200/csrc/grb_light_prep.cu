// grb_light_prep.cu -- LightClusterer::refresh_bindless_prepare for a light list that lives in device memory: frustum
// cull, front-to-back sort and packing into the "cluster-transforms" layout, with the kept count left on the device.
// Compiled with -fmad=false: the per-light arithmetic (grb_light_prep.cuh) must round every operation as the host
// prep does, so the packed bytes are the host's.
//
// Three steps on the caller's stream:
//   1. cull_key_kernel, one thread per input light: visibility and a 33-bit sort key (bit 32 = culled, bits 0..31 the
//      order-preserving code of dot(position, camera_front)) with the light's index as the value;
//   2. cub::DeviceRadixSort::SortPairs over those 33 bits -- stable, so equal keys keep input order, which is the host's
//      by_key_then_input comparator;
//   3. pack_kernel, one thread per slot of GRB_MAX_CLUSTER_LIGHTS: the visible count is where the culled keys begin
//      (a binary search of the sorted keys), and slot s < count packs sorted light s (grb_light_prep_shadowed: with its
//      shadow transform and map; grb_light_prep_shadow_ids: with its transform and this rank's map of its map id).
// The _counted forms read the list's live length on the device: step 1 gives every entry past it the culled key without
// loading it, so steps 2 and 3 are unchanged and never reach those entries.
//
// grb_light_list_to_peers pushes a list's live entries from one rank into every rank's light slot (the protocol is
// grb_peer.cuh's); each receiver then runs the counted prep on its slot, so every rank preps the same bytes.
// grb_light_list_shadowed_to_peers pushes the shadow transforms and map ids with them, and each receiver resolves the ids
// through its own map table (grb_light_prep_shadow_ids): a map pointer is valid on its own rank only, an id anywhere.
#include "grb_common.cuh"
#include "grb_light_prep.cuh"
#include "grb_peer.cuh"

#include <cub/device/device_radix_sort.cuh>

#include <string>
#include <type_traits>

namespace grb
{
namespace
{
constexpr int kMaxInputLights = GRB_MAX_LIGHT_LIST;
constexpr int kPackThreads = 256;

// Counted: only the first lp::live_count(*input_count, lights.count) entries are lights (grb_light_prep[_shadowed]_counted);
// the <false> form keys every entry.
template <bool Counted>
__global__ void __launch_bounds__(256) cull_key_kernel(GrbLightList lights, const int32_t *__restrict__ input_count, GrbLightPrepView view,
                                                       unsigned long long *__restrict__ keys, uint32_t *__restrict__ values)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= lights.count)
		return;
	keys[i] = lp::cull_key(lights, view, i, Counted ? lp::live_count(*input_count, lights.count) : lights.count);
	values[i] = (uint32_t)i;
}

// Shadows: where the shadow tables come from (lp::pack_shadow) -- GrbLightShadowList by map pointer, lp::ShadowIds by map
// id through a table; grb_light_prep runs the lp::NoShadows form, whose code has no shadow part.
template <class Shadows>
__global__ void __launch_bounds__(kPackThreads) pack_kernel(GrbLightList lights, Shadows shadows, GrbLightPrepView view,
                                                           const unsigned long long *__restrict__ keys, const uint32_t *__restrict__ order,
                                                           GrbPositionalLight *__restrict__ records, float *__restrict__ model,
                                                           uint32_t *__restrict__ type_mask, uint2 *__restrict__ z_ranges, float *__restrict__ shadow_transforms,
                                                           const void **__restrict__ shadow_maps, int32_t *__restrict__ count_out)
{
	__shared__ int s_count;
	if (threadIdx.x == 0)
	{
		// the sorted keys hold the visible lights first: the count is the first culled key's index
		int lo = 0, hi = lights.count;
		while (lo < hi)
		{
			const int mid = (lo + hi) >> 1;
			if (keys[mid] >> 32)
				hi = mid;
			else
				lo = mid + 1;
		}
		s_count = min(lo, GRB_MAX_CLUSTER_LIGHTS);
	}
	__syncthreads();
	const int count = s_count;
	const int slots = min(lights.count, GRB_MAX_CLUSTER_LIGHTS);
	const int s = blockIdx.x * blockDim.x + threadIdx.x;
	bool point = false;
	if constexpr (!std::is_same<Shadows, lp::NoShadows>::value)
		if (s < slots)
			lp::pack_shadow(shadows, s < count ? (int)order[s] : -1, s, shadow_transforms, shadow_maps);
	if (s < count)
	{
		const lp::Light L = lp::load_light(lights, (int)order[s]);
		GrbPositionalLight rec;
		float m[12];
		uint32_t zr[2];
		lp::pack(L, view, rec, m, zr);
		records[s] = rec;
		for (int k = 0; k < 12; k++)
			model[12 * s + k] = m[k];
		z_ranges[s] = make_uint2(zr[0], zr[1]);
		point = L.point;
	}
	else if (s < max(slots, 1))
	{
		if (s < slots)
		{
			records[s] = GrbPositionalLight{};
			for (int k = 0; k < 12; k++)
				model[12 * s + k] = 0.0f;
		}
		z_ranges[s] = make_uint2(0xffffffffu, 0u);
	}
	// one type-mask word per warp: every word of the mask is written, zero past the kept lights
	const uint32_t word = __ballot_sync(0xffffffffu, point);
	if ((threadIdx.x & 31) == 0)
		type_mask[s >> 5] = word;
	if (s == 0)
		*count_out = count;
}

// One thread per 16-byte chunk of the capacity's arrays (lp::push_light_chunk: the six of the list, eight with the shadow
// transforms and map ids), then the count word and the publish.
template <int Arrays>
__global__ void __launch_bounds__(256) light_push_kernel(lp::LightPushArrays<Arrays> push, const int32_t *__restrict__ input_count, int capacity,
                                                         PeerTargets targets)
{
	const int live = input_count ? lp::live_count(*input_count, capacity) : capacity;
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	lp::push_light_chunk(push, live, t, targets.data, targets.count);
	if (t == 0)
#pragma unroll
		for (int r = 0; r < GRB_MAX_PEERS; r++)
			if (r < targets.count)
				*reinterpret_cast<int32_t *>(static_cast<uint8_t *>(targets.data[r]) + lp::light_slot_layout().count) = live;
	peer_publish(targets);
}

struct ScratchLayout
{
	size_t keys_in, keys_out, values_in, values_out, temp, temp_bytes, total;
};

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

bool scratch_layout(int n, ScratchLayout &l)
{
	l.temp_bytes = 0;
	if (n > 0 && cub::DeviceRadixSort::SortPairs(nullptr, l.temp_bytes, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
	                                              (const uint32_t *)nullptr, (uint32_t *)nullptr, n, 0, 33) != cudaSuccess)
		return false;
	const size_t n8 = align256((size_t)n * 8), n4 = align256((size_t)n * 4);
	l.keys_in = 0;
	l.keys_out = n8;
	l.values_in = 2 * n8;
	l.values_out = 2 * n8 + n4;
	l.temp = 2 * n8 + 2 * n4;
	l.total = l.temp + align256(l.temp_bytes);
	return true;
}
} // namespace
} // namespace grb

using namespace grb;

extern "C" uint64_t grb_light_prep_scratch_bytes(int32_t max_lights)
{
	ScratchLayout l;
	if (max_lights < 0 || max_lights > kMaxInputLights || !scratch_layout(max_lights, l))
	{
		cudaGetLastError();
		return 0;
	}
	return l.total;
}

namespace
{
// grb_light_prep[_shadowed][_counted] and grb_light_prep_shadow_ids: the checks of grb_light_prep, then the three steps;
// shadows and ids null = the unshadowed pack kernel, input_count null = every entry of the list is a light
int32_t light_prep(const char *fn, const GrbLightList *lights, const int32_t *input_count, const GrbLightShadowList *shadows, const lp::ShadowIds *ids,
                   const GrbLightPrepView *view, GrbPositionalLight *records, float *model, uint32_t *type_mask, uint32_t *z_ranges,
                   float *shadow_transforms, const void **shadow_maps, int32_t *device_count, void *scratch, uint64_t scratch_bytes, void *stream)
{
	if (!lights || !view || !records || !model || !type_mask || !z_ranges || !device_count || lights->count < 0 || lights->count > kMaxInputLights ||
	    (lights->count > 0 && (!lights->color || !lights->position || !lights->is_point || !lights->rotation || !lights->inner_cone ||
	                           !lights->outer_cone || !scratch)))
	{
		set_last_error((std::string(fn) + ": a null pointer or a count outside 0..65536").c_str());
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (shadows && (!shadow_transforms || !shadow_maps || (lights->count > 0 && (!shadows->transforms || !shadows->maps))))
	{
		set_last_error((std::string(fn) + ": a null shadow table").c_str());
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (shadows && (((uintptr_t)shadow_transforms & 7) || ((uintptr_t)shadows->maps & 7) || ((uintptr_t)shadow_maps & 7)))
	{
		set_last_error((std::string(fn) + ": the output transforms, the map array or the output maps are not 8-byte aligned").c_str());
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (ids && (!shadow_transforms || !shadow_maps || (lights->count > 0 && (!ids->ids.transforms || !ids->ids.map_ids))))
	{
		set_last_error((std::string(fn) + ": a null shadow transform or map id array, or a null output table").c_str());
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (ids && (ids->table_size < 0 || ids->table_size > GRB_MAX_LIGHT_LIST || (ids->table_size > 0 && !ids->table)))
	{
		set_last_error((std::string(fn) + ": a map table size outside 0..GRB_MAX_LIGHT_LIST or a null map table").c_str());
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if (ids && (((uintptr_t)shadow_transforms & 7) || ((uintptr_t)ids->table & 7) || ((uintptr_t)shadow_maps & 7) || ((uintptr_t)ids->ids.map_ids & 3)))
	{
		set_last_error((std::string(fn) + ": the output transforms, the map table or the output maps are not 8-byte aligned, or the map ids not 4-byte aligned").c_str());
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if ((uintptr_t)input_count & 3)
	{
		set_last_error((std::string(fn) + ": the input count is not 4-byte aligned").c_str());
		return GRB_ERR_INVALID_ARGUMENT;
	}
	const int n = lights->count;
	ScratchLayout l;
	if (!scratch_layout(n, l))
		return check_launch((std::string(fn) + ": radix sort size").c_str());
	if (scratch_bytes < l.total)
	{
		set_last_error((std::string(fn) + ": scratch smaller than grb_light_prep_scratch_bytes(count)").c_str());
		return GRB_ERR_INVALID_ARGUMENT;
	}
	auto *base = static_cast<uint8_t *>(scratch);
	auto *keys_in = reinterpret_cast<unsigned long long *>(base + l.keys_in), *keys_out = reinterpret_cast<unsigned long long *>(base + l.keys_out);
	auto *values_in = reinterpret_cast<uint32_t *>(base + l.values_in), *values_out = reinterpret_cast<uint32_t *>(base + l.values_out);
	cudaStream_t s = as_stream(stream);
	if (n > 0)
	{
		if (input_count)
			cull_key_kernel<true><<<(n + 255) / 256, 256, 0, s>>>(*lights, input_count, *view, keys_in, values_in);
		else
			cull_key_kernel<false><<<(n + 255) / 256, 256, 0, s>>>(*lights, nullptr, *view, keys_in, values_in);
		int32_t r = check_launch((std::string(fn) + ": cull").c_str());
		if (r != GRB_OK)
			return r;
		size_t temp_bytes = l.temp_bytes;
		if (cub::DeviceRadixSort::SortPairs(base + l.temp, temp_bytes, keys_in, keys_out, values_in, values_out, n, 0, 33, s) != cudaSuccess)
			return check_launch((std::string(fn) + ": sort").c_str());
	}
	auto *ranges = reinterpret_cast<uint2 *>(z_ranges);
	constexpr int blocks = GRB_MAX_CLUSTER_LIGHTS / kPackThreads;
	if (ids)
		pack_kernel<lp::ShadowIds><<<blocks, kPackThreads, 0, s>>>(*lights, *ids, *view, keys_out, values_out, records, model, type_mask, ranges,
		                                                           shadow_transforms, shadow_maps, device_count);
	else if (shadows)
		pack_kernel<GrbLightShadowList><<<blocks, kPackThreads, 0, s>>>(*lights, *shadows, *view, keys_out, values_out, records, model, type_mask, ranges,
		                                                                shadow_transforms, shadow_maps, device_count);
	else
		pack_kernel<lp::NoShadows><<<blocks, kPackThreads, 0, s>>>(*lights, lp::NoShadows{}, *view, keys_out, values_out, records, model, type_mask, ranges,
		                                                           nullptr, nullptr, device_count);
	return check_launch((std::string(fn) + ": pack").c_str());
}
} // namespace

extern "C" int32_t grb_light_prep(const GrbLightList *lights, const GrbLightPrepView *view, GrbPositionalLight *records, float *model, uint32_t *type_mask,
                                  uint32_t *z_ranges, int32_t *device_count, void *scratch, uint64_t scratch_bytes, void *stream)
{
	return light_prep("grb_light_prep", lights, nullptr, nullptr, nullptr, view, records, model, type_mask, z_ranges, nullptr, nullptr, device_count, scratch,
	                  scratch_bytes, stream);
}

extern "C" int32_t grb_light_prep_shadowed(const GrbLightList *lights, const GrbLightShadowList *shadows, const GrbLightPrepView *view,
                                           GrbPositionalLight *records, float *model, uint32_t *type_mask, uint32_t *z_ranges, float *shadow_transforms_out,
                                           const void **shadow_maps_out, int32_t *device_count, void *scratch, uint64_t scratch_bytes, void *stream)
{
	if (!shadows)
	{
		set_last_error("grb_light_prep_shadowed: a null shadow table");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	return light_prep("grb_light_prep_shadowed", lights, nullptr, shadows, nullptr, view, records, model, type_mask, z_ranges, shadow_transforms_out,
	                  shadow_maps_out, device_count, scratch, scratch_bytes, stream);
}

extern "C" int32_t grb_light_prep_counted(const GrbLightList *lights, const int32_t *input_count, const GrbLightPrepView *view, GrbPositionalLight *records,
                                          float *model, uint32_t *type_mask, uint32_t *z_ranges, int32_t *device_count, void *scratch, uint64_t scratch_bytes,
                                          void *stream)
{
	if (!input_count)
	{
		set_last_error("grb_light_prep_counted: a null input count");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	return light_prep("grb_light_prep_counted", lights, input_count, nullptr, nullptr, view, records, model, type_mask, z_ranges, nullptr, nullptr, device_count,
	                  scratch, scratch_bytes, stream);
}

extern "C" int32_t grb_light_prep_shadowed_counted(const GrbLightList *lights, const int32_t *input_count, const GrbLightShadowList *shadows,
                                                   const GrbLightPrepView *view, GrbPositionalLight *records, float *model, uint32_t *type_mask,
                                                   uint32_t *z_ranges, float *shadow_transforms_out, const void **shadow_maps_out, int32_t *device_count,
                                                   void *scratch, uint64_t scratch_bytes, void *stream)
{
	if (!input_count || !shadows)
	{
		set_last_error("grb_light_prep_shadowed_counted: a null input count or shadow table");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	return light_prep("grb_light_prep_shadowed_counted", lights, input_count, shadows, nullptr, view, records, model, type_mask, z_ranges, shadow_transforms_out,
	                  shadow_maps_out, device_count, scratch, scratch_bytes, stream);
}

extern "C" int32_t grb_light_prep_shadow_ids(const GrbLightList *lights, const int32_t *input_count, const GrbLightShadowIdList *ids,
                                             const void *const *map_table, int32_t table_size, const GrbLightPrepView *view, GrbPositionalLight *records,
                                             float *model, uint32_t *type_mask, uint32_t *z_ranges, float *shadow_transforms_out,
                                             const void **shadow_maps_out, int32_t *device_count, void *scratch, uint64_t scratch_bytes, void *stream)
{
	if (!ids)
	{
		set_last_error("grb_light_prep_shadow_ids: a null shadow id list");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	const lp::ShadowIds shadow_ids{ *ids, map_table, table_size };
	return light_prep("grb_light_prep_shadow_ids", lights, input_count, nullptr, &shadow_ids, view, records, model, type_mask, z_ranges,
	                  shadow_transforms_out, shadow_maps_out, device_count, scratch, scratch_bytes, stream);
}

extern "C" int32_t grb_light_slot_layout(void *slot, GrbLightList *out, int32_t **count_out, uint64_t *bytes)
{
	if (!bytes)
	{
		set_last_error("grb_light_slot_layout: a null size pointer");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if ((uintptr_t)slot & 15)
	{
		set_last_error("grb_light_slot_layout: the slot is not 16-byte aligned");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	const lp::LightSlotLayout l = lp::light_slot_layout();
	*bytes = l.bytes;
	auto *base = static_cast<uint8_t *>(slot);
	auto at = [&](int a) { return base ? base + l.array[a] : nullptr; };
	if (out)
	{
		*out = GrbLightList{};
		out->count = GRB_MAX_LIGHT_LIST;
		out->color = reinterpret_cast<const float *>(at(0));
		out->position = reinterpret_cast<const float *>(at(1));
		out->is_point = at(2);
		out->rotation = reinterpret_cast<const float *>(at(3));
		out->inner_cone = reinterpret_cast<const float *>(at(4));
		out->outer_cone = reinterpret_cast<const float *>(at(5));
	}
	if (count_out)
		*count_out = base ? reinterpret_cast<int32_t *>(base + l.count) : nullptr;
	return GRB_OK;
}

namespace
{
// The checks of grb_light_list[_shadowed]_to_peers that need no CUDA call
bool push_arguments(const char *fn, const GrbLightList *lights, const int32_t *input_count, void *const *peer_slots, uint32_t *const *peer_flags,
                    int32_t peer_count, int32_t flag_index, uint32_t epoch, uint32_t *scratch_counter, PeerTargets &targets)
{
	if (!peer_targets_from(fn, peer_slots, peer_flags, peer_count, flag_index, epoch, scratch_counter, targets))
		return false;
	if (!lights || lights->count < 0 || lights->count > GRB_MAX_LIGHT_LIST ||
	    (lights->count > 0 && (!lights->color || !lights->position || !lights->is_point || !lights->rotation || !lights->inner_cone || !lights->outer_cone)))
	{
		set_last_error((std::string(fn) + ": a null light list or array, or a count outside 0..GRB_MAX_LIGHT_LIST").c_str());
		return false;
	}
	if ((uintptr_t)input_count & 3)
	{
		set_last_error((std::string(fn) + ": the input count is not 4-byte aligned").c_str());
		return false;
	}
	for (int r = 0; r < peer_count; r++)
		if ((uintptr_t)peer_slots[r] & 15)
		{
			set_last_error((std::string(fn) + ": a slot is not 16-byte aligned").c_str());
			return false;
		}
	return true;
}

template <int Arrays>
int32_t launch_push(const char *fn, const lp::LightPushArrays<Arrays> &push, const int32_t *input_count, int capacity, const PeerTargets &targets,
                    void *stream)
{
	const unsigned blocks = (unsigned)((push.start[Arrays] + 255) / 256);
	light_push_kernel<Arrays><<<blocks > 0 ? blocks : 1, 256, 0, as_stream(stream)>>>(push, input_count, capacity, targets);
	return check_launch(fn);
}
} // namespace

extern "C" int32_t grb_light_list_to_peers(const GrbLightList *lights, const int32_t *input_count, void *const *peer_slots, uint32_t *const *peer_flags,
                                           int32_t peer_count, int32_t flag_index, uint32_t epoch, uint32_t *scratch_counter, void *stream)
{
	const char *fn = "grb_light_list_to_peers";
	PeerTargets targets;
	if (!push_arguments(fn, lights, input_count, peer_slots, peer_flags, peer_count, flag_index, epoch, scratch_counter, targets))
		return GRB_ERR_INVALID_ARGUMENT;
	return launch_push(fn, lp::light_push(*lights), input_count, lights->count, targets, stream);
}

extern "C" int32_t grb_light_shadow_slot_layout(void *slot, float **transforms, int32_t **map_ids, uint64_t *bytes)
{
	if (!bytes)
	{
		set_last_error("grb_light_shadow_slot_layout: a null size pointer");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	if ((uintptr_t)slot & 15)
	{
		set_last_error("grb_light_shadow_slot_layout: the slot is not 16-byte aligned");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	*bytes = lp::shadow_array_offset(lp::kShadowedLightArrays);
	auto *base = static_cast<uint8_t *>(slot);
	if (transforms)
		*transforms = base ? reinterpret_cast<float *>(base + lp::shadow_array_offset(lp::kLightArrays)) : nullptr;
	if (map_ids)
		*map_ids = base ? reinterpret_cast<int32_t *>(base + lp::shadow_array_offset(lp::kLightArrays + 1)) : nullptr;
	return GRB_OK;
}

extern "C" int32_t grb_light_list_shadowed_to_peers(const GrbLightList *lights, const GrbLightShadowIdList *ids, const int32_t *input_count,
                                                    void *const *peer_slots, uint32_t *const *peer_flags, int32_t peer_count, int32_t flag_index,
                                                    uint32_t epoch, uint32_t *scratch_counter, void *stream)
{
	const char *fn = "grb_light_list_shadowed_to_peers";
	PeerTargets targets;
	if (!push_arguments(fn, lights, input_count, peer_slots, peer_flags, peer_count, flag_index, epoch, scratch_counter, targets))
		return GRB_ERR_INVALID_ARGUMENT;
	if (!ids || (lights->count > 0 && (!ids->transforms || !ids->map_ids)))
	{
		set_last_error("grb_light_list_shadowed_to_peers: a null shadow id list, or null transforms or map ids");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	return launch_push(fn, lp::light_shadow_push(*lights, *ids), input_count, lights->count, targets, stream);
}
