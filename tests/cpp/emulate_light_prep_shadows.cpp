// emulate_light_prep_shadows.cpp -- the shadow part of grb_light_prep_shadowed's pack kernel (lp::pack_shadow in
// granite_b200/csrc/grb_light_prep.cuh) compiled for the CPU (cuda_host_emul.h), run for every slot as the kernel's
// threads do, exported with a C ABI for tests/test_device_lights_shadowed_cpu.py.
#include "cuda_host_emul.h"

#include "../../granite_b200/csrc/grb_light_prep.cuh"

// order: the input index of each kept slot (the radix sort's values), count of them; slots = min(input count, 4096)
extern "C" void emu_pack_shadows(const GrbLightShadowList *shadows, const uint32_t *order, int count, int slots, float *transforms_out,
                                 const void **maps_out)
{
	for (int s = 0; s < slots; s++)
		grb::lp::pack_shadow(*shadows, s < count ? (int)order[s] : -1, s, transforms_out, maps_out);
}
