// gunzip_dev.cuh -- gzip (single or concatenated members) inflated on the GPU: chunked block-start guesses, speculative
// decode with unknown history, chain from the true start, window propagation, exact re-decode into place, parallel CRC-32.
// DESIGN.md section 3c.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

enum { GZ_OK = 0, GZ_REJECT = -2 };

// device memory for the scratch of one inflate (the PAF path hands out its arena, the reads loader plain cudaMalloc)
struct GzMem {
	virtual void *alloc(size_t bytes) = 0;
	virtual void free(void *p) = 0;
	virtual ~GzMem() {}
};

struct GzStats {
	float ms_find, ms_decode, ms_chain, ms_window, ms_resolve, ms_crc; // CUDA-event times of the phases
	uint64_t n_chunks, n_units, n_chain, n_confirmed, n_members, out_len;
	size_t scratch_peak;                                                // bytes of scratch live at once (freed on return)
};

// Inflates the gzip file gz[0, len) (device memory) on `st`.  On success calls out(ctx, n) once for a device buffer of at least
// n bytes, writes the n inflated bytes there and returns GZ_OK with *out_len = n.  Returns GZ_REJECT, having written nothing
// (out may have been called), when the input is not one or more complete, valid gzip members that end exactly at len:
// bad header or header CRC, bad block or code, a distance before the member start, truncation, CRC-32 or ISIZE mismatch,
// trailing bytes.  chunk = 0 picks the default chunk size.  All scratch is freed before it returns.
int gz_inflate_dev(cudaStream_t st, GzMem &mem, const uint8_t *gz, size_t len, char *(*out)(void *ctx, size_t n), void *ctx,
                   size_t *out_len, GzStats *stats = nullptr, size_t chunk = 0);

// the gzip magic (RFC 1952 2.3.1): the loaders take the GPU route only for input that starts with it
static inline bool gz_magic(const void *p, size_t n) { return n >= 2 && ((const uint8_t*)p)[0] == 0x1f && ((const uint8_t*)p)[1] == 0x8b; }
