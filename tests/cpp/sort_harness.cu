// The engine's stable radix sort and top-N pick on their own: two C entry points over gysk::launch_radix_sort and
// gysk::launch_topn_pick (exported from libgysketch.so), so tests/test_gpu_radix_sort.py can hand them torch buffers and a host epoch
// counter it owns. Only the SortTemp fields the sort reads are set. Each returns the launcher's result: its kernel launches, or -1.
#include <cuda_runtime.h>

#include "gysk_kernels.cuh"

static gysk::SortTemp sort_temp(unsigned long long *keys_a, unsigned long long *keys_b, unsigned long long *tile_status, uint32_t max_tiles,
		uint32_t *os_ghist, uint32_t *epoch)
{
	gysk::SortTemp t {};
	t.keys_a = keys_a; t.keys_b = keys_b;
	t.tile_status = tile_status; t.max_tiles = max_tiles;
	t.os_ghist = os_ghist; t.epoch = epoch;
	return t;
}

extern "C" int st_radix_sort(unsigned long long *keys_a, unsigned long long *keys_b, unsigned long long *tile_status, uint32_t max_tiles,
		uint32_t *os_ghist, uint32_t *epoch, const unsigned long long *d_n, uint64_t n_max, int lo, int hi, int *which, cudaStream_t s)
{
	return gysk::launch_radix_sort(sort_temp(keys_a, keys_b, tile_status, max_tiles, os_ghist, epoch), d_n, n_max, lo, hi, which, s);
}

extern "C" int st_topn_pick(unsigned long long *keys_a, unsigned long long *keys_b, unsigned long long *tile_status, uint32_t max_tiles,
		uint32_t *os_ghist, uint32_t *epoch, const unsigned long long *d_n, uint32_t nkeys, const unsigned long long *ids, const uint32_t *hosts,
		uint32_t want, gysk_topn_entry *d_out, unsigned long long *d_slots, cudaStream_t s)
{
	return gysk::launch_topn_pick(sort_temp(keys_a, keys_b, tile_status, max_tiles, os_ghist, epoch), d_n, nkeys, ids, hosts, want, d_out, s, d_slots);
}
