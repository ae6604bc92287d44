// grb_peer.cuh -- the peer-memory exchange of row-sharded frames, shared by every channel (bloom d0 bands, SMAA edge
// rows, TAA history rows, the presented frame; DESIGN.md section 5, "The exchange").
//
// A producing kernel stores its rows into every rank's slot (plain stores to IPC-mapped peer memory over NVLink /
// NVSwitch), then every thread of every CTA calls peer_publish(): the last CTA to arrive at the scratch counter
// resets it and release-stores the frame's epoch into word `flag_index` of every rank's flag array.  A consumer
// acquire-spins on those words with peer_wait(), bounded so that a rank that died cannot hang the GPUs of the others.
#pragma once

#include <cstdio>
#include <cstdlib>

#include "grb_common.cuh"

namespace grb
{
// What a producing kernel needs to reach every rank and to publish its rows there.
struct PeerTargets
{
	void *data[GRB_MAX_PEERS];      // [rank] this frame's slot on that rank; the kernel casts it to its texel type
	uint32_t *flags[GRB_MAX_PEERS]; // [rank] that rank's flag array
	int count;                      // 0: no peers (a kernel that also runs unsharded stores locally)
	int flag_index;                 // this rank's word in every flag array
	uint32_t epoch;
	unsigned *ctas_done; // local scratch counter, 0 between launches
};

__device__ __forceinline__ void store_release_system(uint32_t *p, uint32_t v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t load_acquire_system(const uint32_t *p)
{
	uint32_t v;
	asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}

// Every thread of the CTA must reach this after its last store to a slot.  Each thread's stores are ordered before its
// CTA's arrival; the last CTA to arrive raises this rank's flag on every rank (threadFenceReduction at system scope).
// The flag rises on every rank, also on those that take no row from this one: each consumer waits for all flags.
__device__ __forceinline__ void peer_publish(const PeerTargets &t)
{
	__threadfence_system();
	__syncthreads();
	if (threadIdx.x == 0 && threadIdx.y == 0)
	{
		const unsigned total = gridDim.x * gridDim.y * gridDim.z;
		if (atomicAdd(t.ctas_done, 1u) == total - 1u)
		{
			*t.ctas_done = 0u;
			__threadfence_system();
			for (int r = 0; r < t.count; r++)
				store_release_system(t.flags[r] + t.flag_index, t.epoch);
		}
	}
}

// Spins until rank `rank`'s word of `flags` reaches `epoch` (mod 2^32), at most max_spins times.  On timeout, block 0
// prints (one line per rank however many CTAs wait) and the rank and epoch go to the device error word, which the next
// grb_* call on this device reports (check_launch).
__device__ __forceinline__ void peer_wait(const uint32_t *flags, unsigned rank, uint32_t epoch, uint32_t *error_word, unsigned max_spins)
{
	for (unsigned spins = 0; (int32_t)(load_acquire_system(flags + rank) - epoch) < 0; spins++)
	{
		if (spins > max_spins)
		{
			if (blockIdx.x == 0)
				printf("granite_b200: timed out waiting for rank %d's band of frame %u\n", (int)rank, epoch);
			if (error_word)
			{
				*reinterpret_cast<volatile uint32_t *>(error_word) = (GRB_DEVICE_ERROR_PEER_TIMEOUT << 24) | (rank << 16) | (epoch & 0xffffu);
				__threadfence_system();
			}
			break;
		}
		__nanosleep(128);
	}
}

// The bound of peer_wait: ~4 s by default; GRB_PEER_WAIT_SPINS shortens it (tests of the timeout path).
inline unsigned peer_wait_max_spins()
{
	if (const char *e = getenv("GRB_PEER_WAIT_SPINS"))
		return (unsigned)strtoul(e, nullptr, 10);
	return 1u << 25;
}

// Checks the peer arguments of entry point `fn` and fills `t`; false (with the message set) on a bad argument.
// `flags_only`: no `images` (NULL) -- the kernel writes one rank's slot, which its caller passes on its own
// (grb_present_rows_to_peer), or none (grb_peer_publish).  flag_index must name one of the flag words the ranks wait
// on: a word past them may hold the scratch counter.
inline bool peer_targets_from(const char *fn, void *const *images, uint32_t *const *flags, int32_t count, int32_t flag_index, uint32_t epoch,
                              uint32_t *counter, PeerTargets &t, bool flags_only = false)
{
	char msg[256];
	if ((!images && !flags_only) || !flags || !counter || count < 1 || count > GRB_MAX_PEERS || flag_index < 0 || flag_index >= count)
	{
		snprintf(msg, sizeof(msg), "%s: null pointer, peer_count outside 1..GRB_MAX_PEERS or flag_index outside 0..peer_count-1", fn);
		set_last_error(msg);
		return false;
	}
	t = PeerTargets{};
	for (int r = 0; r < count; r++)
	{
		if ((images && !images[r]) || !flags[r])
		{
			snprintf(msg, sizeof(msg), images ? "%s: null peer pointer" : "%s: null peer flag array", fn);
			set_last_error(msg);
			return false;
		}
		t.data[r] = images ? images[r] : nullptr;
		t.flags[r] = flags[r];
	}
	t.count = count;
	t.flag_index = flag_index;
	t.epoch = epoch;
	t.ctas_done = counter;
	return true;
}

// An empty band still launches one CTA, with nothing to store, so that the flags rise.
inline dim3 peer_grid(int row_count, dim3 grid) { return row_count > 0 ? grid : dim3(1, 1, 1); }
} // namespace grb
