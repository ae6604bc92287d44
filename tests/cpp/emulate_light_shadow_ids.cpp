// emulate_light_shadow_ids.cpp -- shadowed device lights by map id, compiled for the CPU (cuda_host_emul.h): the shadowed
// push of grb_light_list_shadowed_to_peers (lp::light_shadow_push, lp::push_light_chunk) run for every thread of the
// kernel's grid, the shadow part of grb_light_prep_shadow_ids's pack kernel (lp::pack_shadow over lp::ShadowIds) run for
// every slot, and the shadowed slot's layout; all in granite_b200/csrc/grb_light_prep.cuh, exported with a C ABI for
// tests/test_light_shadow_ids_cpu.py.
#include "cuda_host_emul.h"

#include "../../granite_b200/csrc/grb_light_prep.cuh"

// Pushes `lights` (count = the capacity) and `ids` into slots[0..count) with the device count `input_count` (has_count
// 0: every entry live), as the kernel's threads and its thread 0's count-word store do; returns the live length.
extern "C" int emu_shadow_push(const GrbLightList *lights, const GrbLightShadowIdList *ids, int has_count, int32_t input_count, void *const *slots,
                               int count)
{
	const grb::lp::LightShadowPush push = grb::lp::light_shadow_push(*lights, *ids);
	const int live = has_count ? grb::lp::live_count(input_count, lights->count) : lights->count;
	for (int t = 0; t < push.start[grb::lp::kShadowedLightArrays]; t++)
		grb::lp::push_light_chunk(push, live, t, slots, count);
	for (int r = 0; r < count; r++)
		*reinterpret_cast<int32_t *>(static_cast<uint8_t *>(slots[r]) + grb::lp::light_slot_layout().count) = live;
	return live;
}

// The shadow part's offsets: the transforms, the map ids, the shadowed slot's size (3 values)
extern "C" void emu_shadow_slot_layout(uint64_t *out3)
{
	for (int k = 0; k < 3; k++)
		out3[k] = grb::lp::shadow_array_offset(grb::lp::kLightArrays + k);
}

// order: the input index of each kept slot (the radix sort's values), count of them; slots = min(input count, 4096)
extern "C" void emu_pack_shadow_ids(const GrbLightShadowIdList *ids, const void *const *table, int table_size, const uint32_t *order, int count,
                                    int slots, float *transforms_out, const void **maps_out)
{
	const grb::lp::ShadowIds shadows{ *ids, table, table_size };
	for (int s = 0; s < slots; s++)
		grb::lp::pack_shadow(shadows, s < count ? (int)order[s] : -1, s, transforms_out, maps_out);
}
