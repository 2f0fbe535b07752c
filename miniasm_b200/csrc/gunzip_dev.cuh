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

// The compressed bytes of a GzStream: read(off, n, d_dst, st) puts bytes [off, off + n) of the stream into device memory on st
// (the copy may still be in flight on return); false on a read error.
struct GzInput {
	virtual bool read(uint64_t off, size_t n, uint8_t *d_dst, cudaStream_t st) = 0;
	virtual ~GzInput() {}
};

enum { GZ_SMALL = -3 };

// A gzip stream of len compressed bytes inflated a piece at a time, straight into device buffers the caller supplies, with the
// same kernels as gz_inflate_dev run over one compressed segment at a time (DESIGN.md section 3c).  Between fills it keeps the
// absolute bit position of the next unit, whether a member header starts there, the 32 KiB history and how much of it lies
// after the member start, and the raw CRC-32 and length of the member in progress; the stepping decisions are gzstream.cuh's.
//   fill(dst, cap): the next at most cap inflated bytes into dst: their number (> 0), 0 at the end of the stream, GZ_REJECT when
//     the stream is not what gz_inflate_dev accepts (bytes of earlier fills were delivered already), or GZ_SMALL when the next
//     piece alone is longer than cap (*need = its length; nothing was written, a fill with more room goes on).
//   rewind(): back to byte 0.
// A segment takes about cap x (the compressed / inflated ratio so far) compressed bytes (gzs_seg_len), more when one unit cannot
// finish inside it.  Its pass 1 (find + speculative decode) needs no history, so the next segment's runs on a second stream while
// the current one is resolved and the caller parses it.  Scratch of a segment of S compressed bytes in chunks of C (chunk = 0:
// gzs_chunk_for, 4 to 64 KiB) is S + S/C x (64 KiB ring + ~40 B) + 32 KiB per chained unit + 8 B per 16 KiB of output; with the
// next segment's pass 1 beside it (the ring of the current one freed first) at most about S x (2 + 96 KiB / C): 5 S for 32 and
// 64 KiB chunks, 26 S for 4 KiB chunks (segments below 64 MiB); S is about 0.4 x cap for PAF, at most cap + 16 KiB.
struct GzP1;
class GzStream {
public:
	GzStream(cudaStream_t st, GzMem &mem, GzInput &in, uint64_t len, size_t chunk = 0);
	~GzStream();
	int64_t fill(char *dst, size_t cap, size_t *need = nullptr);
	void rewind();
	GzStats sum;                                       // phase times summed over the segments, counts summed, the largest scratch
	uint64_t n_segments = 0, n_grown = 0;              // segments decoded, of them the ones that had to grow
	double ms_read = 0;                                // host wall time of the input reads
private:
	GzP1 *p1_launch(uint64_t bit, uint64_t n, bool hdr, cudaStream_t st);
	int64_t step(GzP1 &p, uint8_t *dst, uint64_t cap, size_t *need);
	void drop_prefetch();
	cudaStream_t st_, st2_;
	GzP1 *pre_ = nullptr;                              // the next segment's pass 1, queued on st2_
	uint64_t next_seg_ = 0;
	GzMem &mem_;
	GzInput &in_;
	uint64_t len_, chunk_, pos_ = 0, in_used_ = 0, out_made_ = 0, need_ = 0;
	bool hdr_ = true, done_ = false;
	uint8_t *hist_;
	uint32_t *valid_;
	unsigned long long *carry_;                        // [0, 1] the member in progress, [2, 3] as the last segment leaves it
	cudaEvent_t ev_[7];
};

// the gzip magic (RFC 1952 2.3.1): the loaders take the GPU route only for input that starts with it
static inline bool gz_magic(const void *p, size_t n) { return n >= 2 && ((const uint8_t*)p)[0] == 0x1f && ((const uint8_t*)p)[1] == 0x8b; }
