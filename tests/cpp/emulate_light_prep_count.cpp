// emulate_light_prep_count.cpp -- the cull step of grb_light_prep_counted (lp::live_count and lp::cull_key in
// granite_b200/csrc/grb_light_prep.cuh) compiled for the CPU (cuda_host_emul.h), run for every entry of the list as the
// cull kernel's threads do, exported with a C ABI for tests/test_device_light_count_cpu.py.
#include "cuda_host_emul.h"

#include "../../granite_b200/csrc/grb_light_prep.cuh"

// keys[i] for i < lights->count with the device count `input_count`; returns the live length the kernel uses
extern "C" int emu_cull_keys(const GrbLightList *lights, const GrbLightPrepView *view, int32_t input_count, unsigned long long *keys)
{
	const int live = grb::lp::live_count(input_count, lights->count);
	for (int i = 0; i < lights->count; i++)
		keys[i] = grb::lp::cull_key(*lights, *view, i, live);
	return live;
}
