// namehash_host.cu -- TEST INFRASTRUCTURE (never linked into the product): the read-name hash of the dictionaries
// (ingest_dev.cuh name_hash, FNV-1a-64 + fmix64) compiled for the host from the very same header, so that
// tests/test_name_collisions_cpu.py can check the numpy restatement that tests/golden/make_name_collisions.py searches with.
#include "../../miniasm_b200/csrc/ingest_dev.cuh"

extern "C" {

// out[i] = name_hash of the bytes [off[i], off[i + 1]) of buf, with `seed`
void nh_hash_many(const char *buf, const uint64_t *off, uint64_t n, uint64_t seed, uint64_t *out)
{
	for (uint64_t i = 0; i < n; ++i) out[i] = name_hash(buf, (uint32_t)off[i], (uint32_t)off[i + 1], seed);
}

}
