// emulate_light_push.cpp -- the push of grb_light_list_to_peers (lp::light_push, lp::push_light_chunk and lp::live_count
// in granite_b200/csrc/grb_light_prep.cuh) compiled for the CPU (cuda_host_emul.h), run for every thread of the kernel's
// grid, exported with a C ABI for tests/test_light_source_rank_cpu.py.
#include "cuda_host_emul.h"

#include "../../granite_b200/csrc/grb_light_prep.cuh"

// Pushes `lights` (count = the capacity) into slots[0..count) with the device count `input_count` (has_count 0: no
// count, every entry live), as the kernel's threads and its thread 0's count-word store do; returns the live length.
extern "C" int emu_push(const GrbLightList *lights, int has_count, int32_t input_count, void *const *slots, int count)
{
	const grb::lp::LightPush push = grb::lp::light_push(*lights);
	const int live = has_count ? grb::lp::live_count(input_count, lights->count) : lights->count;
	for (int t = 0; t < push.start[grb::lp::kLightArrays]; t++)
		grb::lp::push_light_chunk(push, live, t, slots, count);
	for (int r = 0; r < count; r++)
		*reinterpret_cast<int32_t *>(static_cast<uint8_t *>(slots[r]) + grb::lp::light_slot_layout().count) = live;
	return live;
}

// The slot's offsets: count word, the six arrays, the size (8 values)
extern "C" void emu_slot_layout(uint64_t *out8)
{
	const grb::lp::LightSlotLayout l = grb::lp::light_slot_layout();
	out8[0] = l.count;
	for (int a = 0; a < grb::lp::kLightArrays; a++)
		out8[1 + a] = l.array[a];
	out8[7] = l.bytes;
}
