// emulate_light_prep.cpp -- the per-light functions of granite_b200/csrc/grb_light_prep.cuh compiled for the CPU
// (cuda_host_emul.h), applied to every input light, exported with a C ABI for tests/test_device_lights_cpu.py.
#include "cuda_host_emul.h"

#include "../../granite_b200/csrc/grb_light_prep.cuh"

// Per input light i: visibility, the float sort key and its radix code, and the record, model row and Z range the
// pack step would store for it.
extern "C" void emu_light_prep(const GrbLightList *lights, const GrbLightPrepView *view, uint8_t *visible, float *keys, uint32_t *radix,
                               GrbPositionalLight *records, float *model, uint32_t *z_ranges)
{
	for (int i = 0; i < lights->count; i++)
	{
		const grb::lp::Light L = grb::lp::load_light(*lights, i);
		visible[i] = !view->frustum_culling || grb::lp::visible(L, view->planes);
		keys[i] = grb::lp::sort_key(L, view->camera_front);
		radix[i] = grb::lp::radix_key(keys[i]);
		grb::lp::pack(L, *view, records[i], model + 12 * i, z_ranges + 2 * i);
	}
}
