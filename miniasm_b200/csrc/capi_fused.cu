// capi_fused.cu -- fused level of the C ABI (include/miniasm_b200.h, "mab_*"): one device-resident context
// carries the PAF text, the hits, the interval tables and the graphs through all steps of main.c:108-199;
// only counts, the surviving read names and the final structures cross PCIe.
#include "../../include/miniasm_b200.h"
#include "capi_util.cuh"
#include "hit_dev.cuh"
#include "clean_dev.cuh"
#include "gfa_dev.cuh"
#include "dump_dev.cuh"
#include "ugseq_dev.cuh"
#include <pthread.h>
#include "ingest_dev.cuh"
#include "shard_comm.cuh"
#include "gunzip_dev.cuh"
#include <cub/cub.cuh>
#include <map>
#include <string>
#include <zlib.h>
#include <errno.h>
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>

ma_ug_t *mab_ug_download(MabDev &d, DUnitigs &du); // capi_clean.cu
extern "C" sdict_t *sd_from_packed(char *block, size_t block_size, uint32_t n, const uint32_t *len); // host/sdict.c

struct mab_ctx {
	MabDev dev;
	char *d_text = nullptr;
	size_t text_len = 0, text_cap = 0;
	DHits hits;
	DNames names;             // original ids (as assigned by the ingest)
	IngestStats ist;
	uint32_t n_seq = 0;       // current number of reads (after containment removal: the squeezed count)
	uint32_t *orig_id = nullptr; // current id -> original id; null = identity
	DSub *sub = nullptr;      // per current read; null = no read selection ran (-1 -2)
	DGraph sg;
	DUnitigs ug;
	bool have_sg = false, have_ug = false;
	float cov = 40.0f;
	mab_stats_t stats;
	// pinned staging for file loads, and the landing buffers of mab_write_paf / _bed / _sg
	char *pin[2] = {nullptr, nullptr};
	size_t pin_bytes = 0;
	// sharded runs (mab_shard_init): communicator + the packed names of all ranks (names.off indexes it instead of d_text)
	ShardComm sc;
	char *name_text = nullptr;
	char *h_gfa = nullptr;    // pinned landing buffer of mab_write_gfa (grow-only)
	size_t h_gfa_cap = 0;
	// -f reads: the file streams into HBM on its own thread and stream while the graph stages run (mab_reads_prefetch)
	struct ReadsLoad {
		pthread_t tid; bool started = false, joined = false;
		std::string fn;
		int device = 0, rc = 0;
		char *d_text = nullptr;  // cudaMalloc'd by the loader thread (not the arena: that one belongs to the context's own thread)
		size_t len = 0, cap = 0;
	} rl;
};

__global__ void k_sg_len(uint32_t n, const DSub *sub, const uint32_t *slen, const uint32_t *orig, uint32_t *len, uint8_t *del)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		if (sub) len[i] = sub[i].e - (sub[i].s_del & 0x7fffffffu), del[i] = sub[i].s_del >> 31;
		else len[i] = slen[orig ? orig[i] : i], del[i] = 0;
	}
}

__global__ void k_orig_from_map(uint32_t n_old, const int32_t *map, const uint32_t *orig_old, uint32_t *orig_new)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_old; i += gridDim.x * blockDim.x)
		if (map[i] >= 0) orig_new[map[i]] = orig_old ? orig_old[i] : i;
}

__global__ void k_name_sizes(uint32_t n, const uint32_t *orig, const uint32_t *nlen, uint32_t *out)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = nlen[orig ? orig[i] : i] + 1;
}

__global__ void k_name_pack(uint32_t n, const uint32_t *orig, const uint64_t *noff, const uint32_t *nlen, const uint32_t *slen,
                            const char *text, const uint64_t *pos, char *out, uint32_t *out_slen)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const uint32_t o = orig ? orig[i] : i, l = nlen[o];
		const char *src = text + noff[o];
		char *dst = out + pos[i];
		for (uint32_t k = 0; k < l; ++k) dst[k] = src[k];
		dst[l] = 0;
		out_slen[i] = slen[o];
	}
}

struct PhaseTimer { // CUDA-event stopwatch around one step of the fused API (+ host wall clock when MAB_TRACE is set)
	MabDev &d; double *out; cudaEvent_t e0, e1; double w0; const char *name;
	PhaseTimer(MabDev &dev, double *o, const char *nm) : d(dev), out(o), name(nm) { w0 = sys_realtime(); MAB_CUDA(cudaEventCreate(&e0)); MAB_CUDA(cudaEventCreate(&e1)); MAB_CUDA(cudaEventRecord(e0, d.stream)); }
	~PhaseTimer() {
		float ms = 0; MAB_CUDA(cudaEventRecord(e1, d.stream)); MAB_CUDA(cudaEventSynchronize(e1)); MAB_CUDA(cudaEventElapsedTime(&ms, e0, e1)); *out = ms;
		MAB_CUDA(cudaEventDestroy(e0)); MAB_CUDA(cudaEventDestroy(e1));
		if (getenv("MAB_TRACE")) fprintf(stderr, "[T::%s] device %.3f ms, host wall %.3f ms\n", name, ms, (sys_realtime() - w0) * 1e3);
	}
};

extern "C" { static void layout_tail(mab_ctx *c, const ma_opt_t *opt, int stage); }
extern "C" { static void reads_drop(mab_ctx *c); }

static void ctx_drop_graphs(mab_ctx *c)
{
	if (c->have_ug) dg_ug_free(c->dev, c->ug), c->have_ug = false;
	if (c->have_sg) dg_free(c->dev, c->sg), c->have_sg = false;
}

static void ctx_reset_reads(mab_ctx *c)
{
	MabDev &d = c->dev;
	ctx_drop_graphs(c);
	d.free(c->sub), c->sub = nullptr;
	d.free(c->orig_id), c->orig_id = nullptr;
	names_free(d, c->names);
	d.free(c->name_text), c->name_text = nullptr;
	c->hits.n = 0, c->hits.n_seq = 0;
	c->n_seq = 0;
}

// a selection renumbered the reads (map[old] = new id or -1, c->hits.n_seq survivors): carry their original ids over
static void renumber_reads(mab_ctx *c, const int32_t *map, uint32_t n_old)
{
	MabDev &d = c->dev;
	uint32_t *orig_new = mab_alloc<uint32_t>(d, c->hits.n_seq);
	if (n_old) MAB_LAUNCH(d, k_orig_from_map, mab_grid(n_old, 256), 256, 0, n_old, map, c->orig_id, orig_new);
	d.free(c->orig_id);
	c->orig_id = orig_new;
	c->n_seq = c->hits.n_seq;
}

// the default read selection (both rounds, -S 5 and up) on the context's hits
static void select_default(mab_ctx *c, const ma_opt_t *opt, const SelectHooks &hk)
{
	MabDev &d = c->dev;
	const uint32_t n_old = c->n_seq;
	d.free(c->sub);
	c->sub = mab_alloc<DSub>(d, n_old);
	d.trace("select:begin");
	int32_t *map = mab_alloc<int32_t>(d, n_old);
	const SelectParams sp = { opt->min_dp, opt->min_iden, opt->min_span, (int)(opt->max_hang * 1.5), (int)(opt->min_ovlp * .5),
	                          { opt->max_hang, opt->int_frac, opt->min_ovlp } };
	dh_select(d, c->hits, c->sub, sp, map, &c->cov, hk);
	renumber_reads(c, map, n_old);
	d.free(map);
}

extern "C" {

mab_ctx_t *mab_create(int device)
{
	mab_ctx *c = new mab_ctx();
	c->dev.init(device);
	memset(&c->stats, 0, sizeof(c->stats));
	memset(&c->ist, 0, sizeof(c->ist));
	return c;
}

void mab_destroy(mab_ctx_t *c)
{
	if (!c) return;
	MabDev &d = c->dev;
	MAB_CUDA(cudaSetDevice(d.device));
	ctx_reset_reads(c);
	dh_free(d, c->hits);
	d.free(c->d_text);
	d.sync();
	for (int i = 0; i < 2; ++i) if (c->pin[i]) MAB_CUDA(cudaFreeHost(c->pin[i]));
	for (auto &kv : c->sc.ipc_open) cudaIpcCloseMemHandle(kv.second);
	if (c->h_gfa) MAB_CUDA(cudaFreeHost(c->h_gfa));
	reads_drop(c);
	d.destroy();
	delete c;
}

const mab_stats_t *mab_stats(const mab_ctx_t *c)
{
	mab_ctx *m = const_cast<mab_ctx*>(c);
	m->stats.n_kernel_launches = c->dev.n_launch, m->stats.n_lib_calls = c->dev.n_lib;
	return &c->stats;
}

static void text_reserve(mab_ctx *c, size_t len)
{
	if (len <= c->text_cap) return;
	c->dev.free(c->d_text);
	c->text_cap = len + (len >> 3) + 4096;
	c->d_text = (char*)c->dev.alloc(c->text_cap);
	MAB_CUDA(cudaMemsetAsync(c->d_text, 0, c->text_cap, c->dev.stream)); // kernels fetch whole 16-byte words: the bytes after the text are defined
}

/* PAF bytes from host memory to the GPU (one H2D copy; `text` may be pageable or pinned) */
int mab_load_paf_text(mab_ctx_t *c, const char *text, size_t len)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	ctx_reset_reads(c);
	text_reserve(c, len);
	if (len) MAB_CUDA(cudaMemcpyAsync(c->d_text, text, len, cudaMemcpyHostToDevice, c->dev.stream));
	c->text_len = len;
	c->dev.sync();
	return 0;
}

/* ---- gzip input inflated on the GPU (gunzip_dev.cu) ------------------------------------------------------------------ */
struct ArenaMem : GzMem { // the PAF path's scratch: the context's arena (same stream, so frees are immediate)
	MabDev &d;
	explicit ArenaMem(MabDev &dev) : d(dev) {}
	void *alloc(size_t b) override { return d.alloc(b); }
	void free(void *p) override { d.free(p); }
};

struct PlainMem : GzMem { // the reads loader's scratch: cudaMalloc on its own thread
	void *alloc(size_t b) override { void *p; MAB_CUDA(cudaMalloc(&p, b)); return p; }
	void free(void *p) override { MAB_CUDA(cudaFree(p)); }
};

static void gz_trace(const char *what, const GzStats &s, double ms_raw, int rc)
{
	if (!getenv("MAB_TRACE")) return;
	fprintf(stderr, "[T::gunzip] %s rc %d: raw+h2d %.3f find %.3f decode %.3f chain %.3f window %.3f resolve %.3f crc %.3f ms; "
	        "%lu chunks, %lu units, %lu chained, %lu confirmed, %lu members, %lu bytes out, scratch peak %lu\n", what, rc, ms_raw,
	        s.ms_find, s.ms_decode, s.ms_chain, s.ms_window, s.ms_resolve, s.ms_crc, (unsigned long)s.n_chunks, (unsigned long)s.n_units,
	        (unsigned long)s.n_chain, (unsigned long)s.n_confirmed, (unsigned long)s.n_members, (unsigned long)s.out_len, (unsigned long)s.scratch_peak);
}

// the regular file fn when it starts with the gzip magic: an open descriptor and its size; -1 otherwise
static int gz_open_regular(const char *fn, size_t *size)
{
	if (!fn || !strcmp(fn, "-")) return -1;
	const int fd = open(fn, O_RDONLY);
	if (fd < 0) return -1;
	struct stat sb;
	uint8_t mg[2];
	if (fstat(fd, &sb) == 0 && S_ISREG(sb.st_mode) && pread(fd, mg, 2, 0) == 2 && gz_magic(mg, 2)) { *size = (size_t)sb.st_size; return fd; }
	close(fd);
	return -1;
}

// size bytes of fd to dst (device) through two pinned staging buffers of CH bytes: the read of chunk k+1 overlaps the copy of chunk k
static bool read_to_dev(int fd, size_t size, char *dst, char *const pin[2], size_t CH, cudaStream_t st)
{
	cudaEvent_t ev[2];
	for (int i = 0; i < 2; ++i) MAB_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
	size_t done = 0;
	bool ok = true;
	for (int k = 0; ok && done < size; k ^= 1) {
		MAB_CUDA(cudaEventSynchronize(ev[k]));
		const size_t want = size - done < CH ? size - done : CH;
		size_t got = 0;
		while (got < want) {
			const ssize_t r = pread(fd, pin[k] + got, want - got, (off_t)(done + got));
			if (r <= 0) { ok = false; break; }
			got += (size_t)r;
		}
		if (!ok) break;
		MAB_CUDA(cudaMemcpyAsync(dst + done, pin[k], got, cudaMemcpyHostToDevice, st));
		MAB_CUDA(cudaEventRecord(ev[k], st));
		done += got;
	}
	MAB_CUDA(cudaStreamSynchronize(st));
	for (int i = 0; i < 2; ++i) MAB_CUDA(cudaEventDestroy(ev[i]));
	return ok;
}

static void pins_reserve(mab_ctx *c, size_t CH)
{
	if (c->pin_bytes >= CH) return;
	for (int i = 0; i < 2; ++i) { if (c->pin[i]) MAB_CUDA(cudaFreeHost(c->pin[i])); MAB_CUDA(cudaMallocHost(&c->pin[i], CH)); }
	c->pin_bytes = CH;
}

static char *paf_out(void *p, size_t n) // the inflated PAF lands in the context's text buffer
{
	mab_ctx *c = (mab_ctx*)p;
	text_reserve(c, n);
	return c->d_text;
}

// gz[0, len) in device memory (scratch of the arena) -> the context's text; GZ_OK or GZ_REJECT (then the text is empty)
static int paf_inflate(mab_ctx *c, const char *d_gz, size_t len, const char *what, double ms_raw)
{
	ArenaMem am(c->dev);
	GzStats gs;
	memset(&gs, 0, sizeof(gs));
	size_t n = 0;
	const int rc = gz_inflate_dev(c->dev.stream, am, (const uint8_t*)d_gz, len, paf_out, c, &n, &gs);
	c->text_len = rc == GZ_OK ? n : 0;
	if (rc == GZ_OK && c->text_cap > n) MAB_CUDA(cudaMemsetAsync(c->d_text + n, 0, c->text_cap - n, c->dev.stream)); // text_reserve's rule
	c->dev.sync();
	gz_trace(what, gs, ms_raw, rc);
	return rc;
}

/* gzip PAF in host memory, inflated on the GPU: 0, or -2 (nothing loaded) when the GPU decoder rejects the stream */
int mab_load_paf_gz(mab_ctx_t *c, const void *gz, size_t len)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	ctx_reset_reads(c);
	c->text_len = 0;
	if (!gz_magic(gz, len)) return -2;
	const double t0 = sys_realtime();
	char *d_gz = (char*)c->dev.alloc(len);
	MAB_CUDA(cudaMemcpyAsync(d_gz, gz, len, cudaMemcpyHostToDevice, c->dev.stream));
	c->dev.sync();
	const int rc = paf_inflate(c, d_gz, len, "mab_load_paf_gz", (sys_realtime() - t0) * 1e3);
	c->dev.free(d_gz);
	return rc == GZ_OK ? 0 : -2;
}

size_t mab_paf_text(const mab_ctx_t *c, char *dst, size_t cap)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	const size_t n = c->text_len < cap ? c->text_len : cap;
	if (n) MAB_CUDA(cudaMemcpy(dst, c->d_text, n, cudaMemcpyDeviceToHost));
	return c->text_len;
}

/* PAF file (plain or gzip, "-" = stdin) to the GPU through two pinned staging buffers: the read of chunk
 * k+1 overlaps the H2D copy of chunk k.  A regular gzip file crosses compressed and is inflated on the GPU; what the
 * GPU decoder rejects goes through gzread like plain files and stdin.  Returns 0, or -1 if the file cannot be opened. */
int mab_load_paf_file(mab_ctx_t *c, const char *fn)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	const size_t CH = 64u << 20;
	size_t gz_size = 0;
	const int gz_fd = gz_open_regular(fn, &gz_size);
	if (gz_fd >= 0) {
		ctx_reset_reads(c);
		pins_reserve(c, CH);
		const double t0 = sys_realtime();
		char *d_gz = (char*)c->dev.alloc(gz_size);
		int rc = GZ_REJECT;
		if (read_to_dev(gz_fd, gz_size, d_gz, c->pin, CH, c->dev.stream)) rc = paf_inflate(c, d_gz, gz_size, "mab_load_paf_file", (sys_realtime() - t0) * 1e3);
		c->dev.free(d_gz);
		close(gz_fd);
		if (rc == GZ_OK) return 0;
	}
	gzFile fp = fn && strcmp(fn, "-") ? gzopen(fn, "r") : gzdopen(fileno(stdin), "r");
	if (fp == 0) return -1;
	gzbuffer(fp, 1 << 20);
	ctx_reset_reads(c);
	pins_reserve(c, CH);
	struct stat sb;
	size_t guess = 0;
	if (fn && strcmp(fn, "-") && stat(fn, &sb) == 0) guess = (size_t)sb.st_size;
	text_reserve(c, guess ? guess : CH);
	cudaEvent_t ev[2];
	for (int i = 0; i < 2; ++i) MAB_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
	size_t total = 0;
	for (int k = 0;; k ^= 1) {
		MAB_CUDA(cudaEventSynchronize(ev[k])); // the previous copy out of this staging buffer is done
		size_t got = 0;
		while (got < CH) {
			int r = gzread(fp, c->pin[k] + got, (unsigned)((CH - got) < (1u << 30) ? (CH - got) : (1u << 30)));
			if (r <= 0) break;
			got += (size_t)r;
		}
		if (got == 0) break;
		if (total + got > c->text_cap) { // compressed input or stdin: grow the device buffer, keeping what is there
			size_t ncap = (total + got) * 2;
			char *nt = (char*)c->dev.alloc(ncap);
			if (total) MAB_CUDA(cudaMemcpyAsync(nt, c->d_text, total, cudaMemcpyDeviceToDevice, c->dev.stream));
			MAB_CUDA(cudaMemsetAsync(nt + total, 0, ncap - total, c->dev.stream));
			c->dev.free(c->d_text);
			c->d_text = nt, c->text_cap = ncap;
		}
		MAB_CUDA(cudaMemcpyAsync(c->d_text + total, c->pin[k], got, cudaMemcpyHostToDevice, c->dev.stream));
		MAB_CUDA(cudaEventRecord(ev[k], c->dev.stream));
		total += got;
		if (got < CH) break;
	}
	c->dev.sync();
	for (int i = 0; i < 2; ++i) MAB_CUDA(cudaEventDestroy(ev[i]));
	gzclose(fp);
	c->text_len = total;
	return 0;
}

/* Step 1 on the device (hit.c:70-107): parse, name dictionary, mirrored hits, sort */
int mab_ingest(mab_ctx_t *c, int min_span, int min_match, int bi_dir)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	PhaseTimer pt(d, &c->stats.ms_ingest, "mab_ingest");
	ctx_reset_reads(c);
	ingest_paf(d, c->d_text, c->text_len, min_span, min_match, bi_dir, c->hits, c->names, c->ist);
	c->n_seq = c->names.n_seq;
	c->stats.n_lines = c->ist.n_parsed, c->stats.n_hits_stored = c->ist.n_hits, c->stats.n_seq_in = c->ist.n_seq, c->stats.n_name_regrow = c->ist.name_regrow;
	if (!mab_mute && ma_verbose >= 3)
		fprintf(stderr, "[M::%s::%s] read %ld hits; stored %ld hits and %d sequences (%ld bp)\n", "ma_hit_read", sys_timestamp(),
				(long)c->ist.n_parsed, (long)c->ist.n_hits, (int)c->ist.n_seq, (long)c->ist.tot_len);
	return 0;
}

/* mab_load_paf_text + mab_ingest in one call, overlapped: chunk k of the text is scanned for line starts and parsed (store filter,
 * dictionary) while chunk k+1 crosses PCIe on a second stream; when the last byte lands only the id ranking, the hit emission and the
 * sort are left.  `text` may be pageable or pinned (pinned overlaps fully). */
int mab_load_ingest_text(mab_ctx_t *c, const char *text, size_t len, int min_span, int min_match, int bi_dir)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	ctx_reset_reads(c);
	text_reserve(c, len);
	c->text_len = len;
	PhaseTimer pt(d, &c->stats.ms_ingest, "mab_load_ingest_text");
	ingest_paf_stream(d, c->d_text, text, len, min_span, min_match, bi_dir, c->hits, c->names, c->ist);
	c->n_seq = c->names.n_seq;
	c->stats.n_lines = c->ist.n_parsed, c->stats.n_hits_stored = c->ist.n_hits, c->stats.n_seq_in = c->ist.n_seq, c->stats.n_name_regrow = c->ist.name_regrow;
	if (!mab_mute && ma_verbose >= 3)
		fprintf(stderr, "[M::%s::%s] read %ld hits; stored %ld hits and %d sequences (%ld bp)\n", "ma_hit_read", sys_timestamp(),
				(long)c->ist.n_parsed, (long)c->ist.n_hits, (int)c->ist.n_seq, (long)c->ist.tot_len);
	return 0;
}

/* ---- Step 1 in windows: the text never becomes resident (ingest_paf_windowed, DESIGN.md 3d) ---------------------------- */
static int ingest_windowed(mab_ctx *c, const TextSource &src, size_t window_bytes, size_t size_hint, int min_span, int min_match, int bi_dir)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	PhaseTimer pt(d, &c->stats.ms_ingest, "mab_ingest_windowed");
	ctx_reset_reads(c);
	d.free(c->d_text), c->d_text = nullptr, c->text_len = c->text_cap = 0; // a text loaded earlier is given up: this ingest keeps names, not text
	if (!ingest_paf_windowed(d, src, window_bytes ? window_bytes : (size_t)256 << 20, size_hint, min_span, min_match, bi_dir, c->hits, c->names, &c->name_text, c->ist))
		return -1;
	c->n_seq = c->names.n_seq;
	c->stats.n_lines = c->ist.n_parsed, c->stats.n_hits_stored = c->ist.n_hits, c->stats.n_seq_in = c->ist.n_seq, c->stats.n_name_regrow = c->ist.name_regrow;
	if (!mab_mute && ma_verbose >= 3)
		fprintf(stderr, "[M::%s::%s] read %ld hits; stored %ld hits and %d sequences (%ld bp)\n", "ma_hit_read", sys_timestamp(),
				(long)c->ist.n_parsed, (long)c->ist.n_hits, (int)c->ist.n_seq, (long)c->ist.tot_len);
	return 0;
}

int mab_ingest_windowed(mab_ctx_t *c, const mab_text_source_t *src, size_t window_bytes, int min_span, int min_match, int bi_dir)
{
	const TextSource ts = { src->read, src->rewind, src->ud };
	return ingest_windowed(c, ts, window_bytes, 0, min_span, min_match, bi_dir);
}

struct FileSource { int fd; gzFile gz; }; // a plain file is read and sought directly, a gzip file through zlib on the host

static size_t file_read(void *ud, char *dst, size_t cap)
{
	FileSource *f = (FileSource*)ud;
	if (f->gz) { const int r = gzread(f->gz, dst, (unsigned)(cap < (1u << 30) ? cap : (1u << 30))); return r > 0 ? (size_t)r : 0; }
	ssize_t r;
	do r = read(f->fd, dst, cap); while (r < 0 && errno == EINTR);
	return r > 0 ? (size_t)r : 0;
}

static int file_rewind(void *ud)
{
	FileSource *f = (FileSource*)ud;
	return f->gz ? gzrewind(f->gz) : lseek(f->fd, 0, SEEK_SET) == 0 ? 0 : -1;
}

int mab_ingest_file_windowed(mab_ctx_t *c, const char *fn, size_t window_bytes, int min_span, int min_match, int bi_dir)
{
	FileSource f = { fn && strcmp(fn, "-") ? open(fn, O_RDONLY) : dup(fileno(stdin)), nullptr };
	if (f.fd < 0) return -1;
	struct stat sb;
	uint8_t mg[2];
	size_t hint = fstat(f.fd, &sb) == 0 && S_ISREG(sb.st_mode) ? (size_t)sb.st_size : 0;
	if (hint && pread(f.fd, mg, 2, 0) == 2 && gz_magic(mg, 2)) {
		f.gz = gzdopen(f.fd, "r");
		if (f.gz == 0) { close(f.fd); return -1; }
		gzbuffer(f.gz, 1 << 20);
		hint *= 4;                                   // (a guess at the inflated size: it only sizes the first dictionary)
	}
	const TextSource ts = { file_read, file_rewind, &f };
	const int rc = ingest_windowed(c, ts, window_bytes, hint, min_span, min_match, bi_dir);
	if (f.gz) gzclose(f.gz); else close(f.fd);
	return rc < 0 ? -2 : 0;
}

size_t mab_mem_peak(mab_ctx_t *c, int reset)
{
	const size_t p = c->dev.arena.peak;
	if (reset) c->dev.arena.peak = c->dev.arena.in_use;
	return p;
}

size_t mab_mem_free(mab_ctx_t *c)
{
	size_t fr = 0, tot = 0;
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MAB_CUDA(cudaMemGetInfo(&fr, &tot));
	return fr + (c->dev.arena.reserved - c->dev.arena.in_use);
}

/* -R (main.c:110-113 + hit.c:38-68,86): Step 0 and Step 1 in one pass over the text that is already in HBM.  Prints the
 * reference's two log lines and its Step-1 banner in the reference's order. */
int mab_ingest_nocont(mab_ctx_t *c, int min_span, int min_match, int bi_dir, int max_hang, float int_frac)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	PhaseTimer pt(d, &c->stats.ms_ingest, "mab_ingest_nocont");
	ctx_reset_reads(c);
	NoContParams nc = { max_hang, int_frac };
	ingest_paf(d, c->d_text, c->text_len, min_span, min_match, bi_dir, c->hits, c->names, c->ist, &nc);
	c->n_seq = c->names.n_seq;
	c->stats.n_lines = c->ist.n_parsed, c->stats.n_hits_stored = c->ist.n_hits, c->stats.n_seq_in = c->ist.n_seq, c->stats.n_name_regrow = c->ist.name_regrow;
	if (!mab_mute && ma_verbose >= 3) fprintf(stderr, "[M::%s::%s] dropped %d contained reads\n", "ma_hit_no_cont", sys_timestamp(), (int)c->ist.n_dropped);
	if (!mab_mute) fprintf(stderr, "[M::main] ===> Step 1: reading read mappings <===\n");
	if (!mab_mute && ma_verbose >= 3)
		fprintf(stderr, "[M::%s::%s] read %ld hits; stored %ld hits and %d sequences (%ld bp)\n", "ma_hit_read", sys_timestamp(),
				(long)c->ist.n_parsed, (long)c->ist.n_hits, (int)c->ist.n_seq, (long)c->ist.tot_len);
	return 0;
}

/* Alternative to mab_ingest: hits parsed elsewhere (e.g. ma_hit_read with an exclusion dictionary, -R) */
int mab_load_hits(mab_ctx_t *c, const ma_hit_t *a, size_t n, const sdict_t *dict)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	ctx_reset_reads(c);
	dh_reserve(d, c->hits, n ? n : 1);
	c->hits.n = n, c->hits.n_seq = dict->n_seq;
	if (n) MAB_CUDA(cudaMemcpyAsync(c->hits.a, a, n * sizeof(DHit), cudaMemcpyHostToDevice, d.stream));
	// names live on the host in this mode: pack them into the text buffer so that the export path is the same
	size_t bytes = 0;
	for (uint32_t i = 0; i < dict->n_seq; ++i) bytes += strlen(dict->seq[i].name) + 1;
	char *pack = (char*)malloc(bytes ? bytes : 1);
	uint64_t *off = (uint64_t*)malloc((dict->n_seq ? dict->n_seq : 1) * 8);
	uint32_t *nl = (uint32_t*)malloc((dict->n_seq ? dict->n_seq : 1) * 4), *sl = (uint32_t*)malloc((dict->n_seq ? dict->n_seq : 1) * 4);
	bytes = 0;
	for (uint32_t i = 0; i < dict->n_seq; ++i) {
		size_t l = strlen(dict->seq[i].name);
		memcpy(pack + bytes, dict->seq[i].name, l + 1);
		off[i] = bytes, nl[i] = (uint32_t)l, sl[i] = dict->seq[i].len;
		bytes += l + 1;
	}
	text_reserve(c, bytes);
	c->text_len = bytes;
	DNames &nm = c->names;
	nm.n_seq = dict->n_seq;
	nm.off = mab_alloc<uint64_t>(d, nm.n_seq); nm.nlen = mab_alloc<uint32_t>(d, nm.n_seq); nm.slen = mab_alloc<uint32_t>(d, nm.n_seq);
	if (bytes) MAB_CUDA(cudaMemcpyAsync(c->d_text, pack, bytes, cudaMemcpyHostToDevice, d.stream));
	if (nm.n_seq) {
		MAB_CUDA(cudaMemcpyAsync(nm.off, off, (size_t)nm.n_seq * 8, cudaMemcpyHostToDevice, d.stream));
		MAB_CUDA(cudaMemcpyAsync(nm.nlen, nl, (size_t)nm.n_seq * 4, cudaMemcpyHostToDevice, d.stream));
		MAB_CUDA(cudaMemcpyAsync(nm.slen, sl, (size_t)nm.n_seq * 4, cudaMemcpyHostToDevice, d.stream));
	}
	d.sync();
	free(pack); free(off); free(nl); free(sl);
	c->n_seq = dict->n_seq;
	c->stats.n_hits_stored = n, c->stats.n_seq_in = dict->n_seq, c->stats.n_name_regrow = 0;
	return 0;
}

/* Steps 2-3 (main.c:119-142): read selection.  `stage` has the meaning of the reference's -S. */
int mab_select(mab_ctx_t *c, const ma_opt_t *opt, int no_first, int no_second, int stage)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	DHits &h = c->hits;
	PhaseTimer pt(d, &c->stats.ms_select, "mab_select");
	ctx_drop_graphs(c);
	dh_hits_dense(d, h);   // a selection again: the step functions need the dense array
	auto step3_banner = [] { if (!mab_mute && ma_verbose >= 1) fprintf(stderr, "[M::main] ===> Step 3: 2-pass (fine) read selection <===\n"); };
	if (!no_first && !no_second && stage >= 5) { // the whole selection: per-read passes over the hit buckets
		if (!mab_mute && ma_verbose >= 1) fprintf(stderr, "[M::main] ===> Step 2: 1-pass (crude) read selection <===\n");
		select_default(c, opt, { step3_banner });
		c->stats.n_hits_final = h.n, c->stats.n_seq_final = c->n_seq;
		d.sync();
		return 0;
	}
	if (!no_first) {
		if (!mab_mute && ma_verbose >= 1) fprintf(stderr, "[M::main] ===> Step 2: 1-pass (crude) read selection <===\n");
		if (stage >= 2) {
			d.free(c->sub);
			c->sub = mab_alloc<DSub>(d, c->n_seq);
			d.trace("select:begin");
			dh_sub(d, h, opt->min_dp, opt->min_iden, 0, c->sub);
			d.trace("select:sub1");
			dh_cut(d, h, c->sub, opt->min_span);
			if (stage >= 3) dh_flt(d, h, c->sub, (int)(opt->max_hang * 1.5), (int)(opt->min_ovlp * .5), &c->cov);
			d.trace("select:cut1(+flt)");
		}
	}
	if (!no_second) {
		step3_banner();
		if (stage >= 4) {
			DSub *sub2 = mab_alloc<DSub>(d, c->n_seq);
			d.trace("select:flt");
			dh_sub(d, h, opt->min_dp, opt->min_iden, opt->min_span / 2, sub2);
			d.trace("select:sub2");
			dh_cut(d, h, sub2, opt->min_span);
			if (!no_first && c->sub) { dh_sub_merge(d, c->n_seq, c->sub, sub2); d.free(sub2); }
			else { d.free(c->sub); c->sub = sub2; }
		}
		if (stage >= 5 && c->sub) {
			const uint32_t n_old = c->n_seq;
			int32_t *map = mab_alloc<int32_t>(d, n_old);
			HitArcParams p = { opt->max_hang, opt->int_frac, opt->min_ovlp };
			dh_contained(d, h, c->sub, nullptr, p, map);
			renumber_reads(c, map, n_old);
			d.free(map);
			d.trace("select:contained");
		}
	}
	c->stats.n_hits_final = h.n, c->stats.n_seq_final = c->n_seq;
	d.sync();
	return 0;
}

/* Step 4 (main.c:155-188): graph construction and cleaning.  stage as in -S (5 = raw graph ... 11 = all). */
int mab_layout(mab_ctx_t *c, const ma_opt_t *opt, int stage)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	PhaseTimer pt(d, &c->stats.ms_layout, "mab_layout");
	ctx_drop_graphs(c);
	uint32_t *len = mab_alloc<uint32_t>(d, c->n_seq);
	uint8_t *del = mab_alloc<uint8_t>(d, c->n_seq);
	if (c->n_seq) MAB_LAUNCH(d, k_sg_len, mab_grid(c->n_seq, 256), 256, 0, c->n_seq, c->sub, c->names.slen, c->orig_id, len, del);
	HitArcParams p = { opt->max_hang, opt->int_frac, opt->min_ovlp };
	c->hits.n_seq = c->n_seq;
	d.trace("layout:begin");
	dh_sg_gen(d, c->hits, len, del, p, c->sg);
	d.trace("layout:sg_gen");
	c->have_sg = true;
	d.free(len); d.free(del);
	DGraph &g = c->sg;
	c->stats.n_arc_sg = g.n_arc;
	if (stage >= 6) {
		if (!mab_mute && ma_verbose >= 1) fprintf(stderr, "[M::main] ===> Step 4.1: transitive reduction <===\n");
		dg_del_trans(d, g, (uint32_t)opt->gap_fuzz);
		c->stats.n_arc_trans_in = g_del_trans_stats.n_arc_in, c->stats.n_reduced = g_del_trans_stats.n_reduced;
		c->stats.trans_inner = g_del_trans_stats.inner_iters, c->stats.ms_del_trans_kernel = g_del_trans_stats.kernel_ms;
		d.trace("layout:del_trans+cleanup+symm");
	}
	layout_tail(c, opt, stage);
	return 0;
}

/* main.c:160-188: the passes after transitive reduction, on the (replicated) reduced graph */
static void layout_tail(mab_ctx *c, const ma_opt_t *opt, int stage)
{
	MabDev &d = c->dev;
	DGraph &g = c->sg;
	g_clean_stats = CleanStats();                          // mab_clean_totals counts the passes of this layout
	if (stage >= 7) {
		if (!mab_mute && ma_verbose >= 1) fprintf(stderr, "[M::main] ===> Step 4.2: initial tip cutting and bubble popping <===\n");
		dg_cut_tip(d, g, opt->max_ext);
		dg_pop_bubble(d, g, opt->bub_dist);
	}
	if (stage >= 9) {
		if (!mab_mute && ma_verbose >= 1) fprintf(stderr, "[M::main] ===> Step 4.3: cutting short overlaps (%d rounds in total) <===\n", opt->n_rounds + 1);
		for (int i = 0; i <= opt->n_rounds; ++i) {
			float r = opt->min_ovlp_drop_ratio + (opt->max_ovlp_drop_ratio - opt->min_ovlp_drop_ratio) / opt->n_rounds * i;
			if (dg_del_short(d, g, r) != 0) {
				dg_cut_tip(d, g, opt->max_ext);
				dg_pop_bubble(d, g, opt->bub_dist);
			}
		}
	}
	if (stage >= 10) {
		if (!mab_mute && ma_verbose >= 1) fprintf(stderr, "[M::main] ===> Step 4.4: removing short internal sequences and bi-loops <===\n");
		dg_cut_internal(d, g, 1);
		dg_cut_biloop(d, g, opt->max_ext);
		dg_cut_tip(d, g, opt->max_ext);
		dg_pop_bubble(d, g, opt->bub_dist);
	}
	if (stage >= 11) {
		if (!mab_mute && ma_verbose >= 1) fprintf(stderr, "[M::main] ===> Step 4.5: aggressively cutting short overlaps <===\n");
		if (dg_del_short(d, g, opt->final_ovlp_drop_ratio) != 0) {
			dg_cut_tip(d, g, opt->max_ext);
			dg_pop_bubble(d, g, opt->bub_dist);
		}
	}
	c->stats.n_arc_final = g.n_arc;
	d.sync();
	d.trace("layout:cleaning passes");
}

/* Step 5 (asm.c:121-210) */
int mab_unitigs(mab_ctx_t *c)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	if (!c->have_sg) return -1;
	PhaseTimer pt(c->dev, &c->stats.ms_unitigs, "mab_unitigs");
	if (c->have_ug) dg_ug_free(c->dev, c->ug), c->have_ug = false;
	dg_ug_gen(c->dev, c->sg, c->ug);
	c->have_ug = true;
	c->stats.n_utg = c->ug.n_utg;
	c->dev.sync();
	return 0;
}

/* ---- exports: reference-compatible host structures, owned by the caller -------------------------------- */

sdict_t *mab_export_dict(mab_ctx_t *c)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	sdict_t *dict = sd_init();
	const uint32_t n = c->n_seq;
	if (n == 0) return dict;
	uint32_t *sz = mab_alloc<uint32_t>(d, n), *d_slen = mab_alloc<uint32_t>(d, n);
	uint64_t *pos = mab_alloc<uint64_t>(d, (size_t)n + 1);
	MAB_LAUNCH(d, k_name_sizes, mab_grid(n, 256), 256, 0, n, c->orig_id, c->names.nlen, sz);
	size_t tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tb, sz, pos, (int)n, d.stream);
	void *tmp = d.tmp(tb);
	cub::DeviceScan::ExclusiveSum(tmp, tb, sz, pos, (int)n, d.stream);
	++d.n_lib;
	uint64_t last_pos; uint32_t last_sz;
	MAB_CUDA(cudaMemcpyAsync(&last_pos, pos + n - 1, 8, cudaMemcpyDeviceToHost, d.stream));
	MAB_CUDA(cudaMemcpyAsync(&last_sz, sz + n - 1, 4, cudaMemcpyDeviceToHost, d.stream));
	d.sync();
	const size_t bytes = last_pos + last_sz;
	char *d_pack = (char*)d.alloc(bytes), *pack = (char*)malloc(bytes);
	uint32_t *slen = (uint32_t*)malloc((size_t)n * 4);
	MAB_LAUNCH(d, k_name_pack, mab_grid(n, 256), 256, 0, n, c->orig_id, c->names.off, c->names.nlen, c->names.slen, c->name_text ? c->name_text : c->d_text, pos, d_pack, d_slen);
	MAB_CUDA(cudaMemcpyAsync(pack, d_pack, bytes, cudaMemcpyDeviceToHost, d.stream));
	MAB_CUDA(cudaMemcpyAsync(slen, d_slen, (size_t)n * 4, cudaMemcpyDeviceToHost, d.stream));
	d.sync();
	sd_destroy(dict);
	dict = sd_from_packed(pack, bytes, n, slen); // takes `pack`; the hash index is built only if a name is looked up
	free(slen);
	d.free(sz); d.free(d_slen); d.free(pos); d.free(d_pack);
	d.sync();
	return dict;
}

ma_sub_t *mab_export_sub(mab_ctx_t *c)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	if (!c->sub) return 0;
	ma_sub_t *s = (ma_sub_t*)calloc(c->n_seq ? c->n_seq : 1, sizeof(ma_sub_t));
	if (c->n_seq) MAB_CUDA(cudaMemcpyAsync(s, c->sub, (size_t)c->n_seq * sizeof(DSub), cudaMemcpyDeviceToHost, c->dev.stream));
	c->dev.sync();
	return s;
}

ma_hit_t *mab_export_hits(mab_ctx_t *c, size_t *n)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	dh_hits_dense(c->dev, c->hits);
	ma_hit_t *a = (ma_hit_t*)malloc((c->hits.n ? c->hits.n : 1) * sizeof(ma_hit_t));
	if (c->hits.n) MAB_CUDA(cudaMemcpyAsync(a, c->hits.a, c->hits.n * sizeof(DHit), cudaMemcpyDeviceToHost, c->dev.stream));
	c->dev.sync();
	*n = c->hits.n;
	return a;
}

asg_t *mab_export_sg(mab_ctx_t *c)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	if (!c->have_sg) return 0;
	asg_t *g = asg_init();
	g->n_seq = c->sg.n_seq, g->m_seq = c->sg.n_seq ? c->sg.n_seq : 1;
	g->seq = (asg_seq_t*)malloc((size_t)g->m_seq * sizeof(asg_seq_t));
	g->m_arc = c->sg.n_arc ? c->sg.n_arc : 1;
	g->arc = (asg_arc_t*)malloc((size_t)g->m_arc * sizeof(asg_arc_t));
	mab_graph_download(c->dev, c->sg, g);
	return g;
}

ma_ug_t *mab_export_ug(mab_ctx_t *c)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	if (!c->have_ug) return 0;
	return mab_ug_download(c->dev, c->ug);
}

float mab_coverage(const mab_ctx_t *c) { return c->cov; }

/* ma_ug_print(mab_export_ug, mab_export_dict, mab_export_sub, fp) without the host structs: the text is formatted on
 * the GPU (gfa_dev.cu), copied down once and written with one fwrite.  Unitig sequences are not part of it ("*").
 * Returns the number of bytes written, -1 if mab_unitigs has not run. */
long mab_write_gfa(mab_ctx_t *c, FILE *fp)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	if (!c->have_ug) return -1;
	MabDev &d = c->dev;
	if (!c->ug.g.has_idx) dg_arc_index(d, c->ug.g); // the x lines print the arc counts of both unitig ends (asm.c:110-112)
	char *d_txt = nullptr;
	const size_t n = dg_gfa_text(d, c->ug, c->orig_id, c->names.off, c->names.nlen, c->name_text ? c->name_text : c->d_text, c->sub, &d_txt);
	if (n) {
		if (n > c->h_gfa_cap) {
			if (c->h_gfa) MAB_CUDA(cudaFreeHost(c->h_gfa));
			c->h_gfa_cap = n + (n >> 2) + (1 << 20);
			MAB_CUDA(cudaHostAlloc((void**)&c->h_gfa, c->h_gfa_cap, cudaHostAllocDefault));
		}
		MAB_CUDA(cudaMemcpyAsync(c->h_gfa, d_txt, n, cudaMemcpyDeviceToHost, d.stream));
		d.sync();
		if (fwrite(c->h_gfa, 1, n, fp) != n) { fprintf(stderr, "[E::miniasm_b200] short write of the GFA text\n"); exit(74); }
	}
	d.free(d_txt);
	d.sync();
	return (long)n;
}

/* -p paf | bed | sg: the text formatted on the GPU (dump_dev.cu) and written in chunks; names come from the context's name table
 * (name_text after a sharded ingest), intervals from its table of the current reads */
static long write_dump(mab_ctx *c, DumpKind kind, uint64_t n_rec, FILE *fp)
{
	const DumpView v{{c->orig_id, c->names.off, c->names.nlen, c->name_text ? c->name_text : c->d_text, c->sub}, c->hits.a, c->sg.arc};
	return (long)dg_dump_write(c->dev, kind, v, n_rec, fp, c->pin, c->pin_bytes);
}

/* print_hits (main.c:21-30) of the current hits; -1 (nothing written) when no read selection ran */
long mab_write_paf(mab_ctx_t *c, FILE *fp)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	if (!c->sub) return -1;
	dh_hits_dense(c->dev, c->hits);
	return write_dump(c, DUMP_PAF, c->hits.n, fp);
}

/* print_subs (main.c:13-19) of the current reads; -1 (nothing written) when no read selection ran */
long mab_write_bed(mab_ctx_t *c, FILE *fp)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	if (!c->sub) return -1;
	return write_dump(c, DUMP_BED, c->n_seq, fp);
}

/* ma_sg_print (asm.c:41-55) of the string graph; -1 before mab_layout */
long mab_write_sg(mab_ctx_t *c, FILE *fp)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	if (!c->have_sg) return -1;
	return write_dump(c, DUMP_SG, c->sg.n_arc, fp);
}

/* ---- -f reads (ma_ug_seq, asm.c:236-290) ------------------------------------------------------------------------------- */
static char *reads_out(void *p, size_t n) // the inflated reads land in a buffer of the loader's own
{
	mab_ctx::ReadsLoad *rl = (mab_ctx::ReadsLoad*)p;
	rl->cap = n + 4096;
	MAB_CUDA(cudaMalloc(&rl->d_text, rl->cap));
	return rl->d_text;
}

// a regular gzip reads file: compressed bytes to HBM, inflated there; false (nothing kept) when the GPU decoder rejects it
static bool reads_gunzip(mab_ctx::ReadsLoad *rl, int fd, size_t size, size_t CH)
{
	cudaStream_t st;
	char *pin[2], *d_gz;
	MAB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
	for (int i = 0; i < 2; ++i) MAB_CUDA(cudaMallocHost(&pin[i], CH));
	MAB_CUDA(cudaMalloc(&d_gz, size));
	const double t0 = sys_realtime();
	int rc = GZ_REJECT;
	GzStats gs;
	memset(&gs, 0, sizeof(gs));
	if (read_to_dev(fd, size, d_gz, pin, CH, st)) {
		const double ms_raw = (sys_realtime() - t0) * 1e3;
		PlainMem pm;
		size_t n = 0;
		rc = gz_inflate_dev(st, pm, (const uint8_t*)d_gz, size, reads_out, rl, &n, &gs);
		if (rc == GZ_OK) { rl->len = n; MAB_CUDA(cudaMemsetAsync(rl->d_text + n, 0, rl->cap - n, st)); }
		MAB_CUDA(cudaStreamSynchronize(st));
		gz_trace("reads_loader", gs, ms_raw, rc);
	}
	if (rc != GZ_OK && rl->d_text) { MAB_CUDA(cudaFree(rl->d_text)); rl->d_text = nullptr, rl->len = rl->cap = 0; }
	MAB_CUDA(cudaFree(d_gz));
	for (int i = 0; i < 2; ++i) MAB_CUDA(cudaFreeHost(pin[i]));
	MAB_CUDA(cudaStreamDestroy(st));
	return rc == GZ_OK;
}

static void *reads_loader(void *p) // file -> pinned double buffer -> HBM, on a stream of its own
{
	mab_ctx::ReadsLoad *rl = (mab_ctx::ReadsLoad*)p;
	const size_t CH = 32u << 20;
	cudaStream_t st;
	char *pin[2];
	cudaEvent_t ev[2];
	MAB_CUDA(cudaSetDevice(rl->device));
	size_t gz_size = 0;
	const int gz_fd = gz_open_regular(rl->fn.c_str(), &gz_size);
	if (gz_fd >= 0) {
		const bool ok = reads_gunzip(rl, gz_fd, gz_size, CH);
		close(gz_fd);
		if (ok) return 0;
	}
	gzFile fp = rl->fn != "-" ? gzopen(rl->fn.c_str(), "r") : gzdopen(fileno(stdin), "r");
	if (fp == 0) { rl->rc = -1; return 0; }
	gzbuffer(fp, 1 << 20);
	MAB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
	for (int i = 0; i < 2; ++i) { MAB_CUDA(cudaMallocHost(&pin[i], CH)); MAB_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming)); }
	struct stat sb;
	size_t guess = 0;
	if (rl->fn != "-" && stat(rl->fn.c_str(), &sb) == 0) guess = (size_t)sb.st_size;
	rl->cap = (guess ? guess : CH) + 4096;
	MAB_CUDA(cudaMalloc(&rl->d_text, rl->cap));
	for (int k = 0;; k ^= 1) {
		MAB_CUDA(cudaEventSynchronize(ev[k]));
		size_t got = 0;
		while (got < CH) {
			int r = gzread(fp, pin[k] + got, (unsigned)(CH - got));
			if (r <= 0) break;
			got += (size_t)r;
		}
		if (got == 0) break;
		if (rl->len + got + 64 > rl->cap) { // compressed input: grow, keeping what is there
			size_t ncap = (rl->len + got) * 2 + 4096;
			char *nt;
			MAB_CUDA(cudaStreamSynchronize(st));
			MAB_CUDA(cudaMalloc(&nt, ncap));
			if (rl->len) MAB_CUDA(cudaMemcpyAsync(nt, rl->d_text, rl->len, cudaMemcpyDeviceToDevice, st));
			MAB_CUDA(cudaStreamSynchronize(st));
			MAB_CUDA(cudaFree(rl->d_text));
			rl->d_text = nt, rl->cap = ncap;
		}
		MAB_CUDA(cudaMemcpyAsync(rl->d_text + rl->len, pin[k], got, cudaMemcpyHostToDevice, st));
		MAB_CUDA(cudaEventRecord(ev[k], st));
		rl->len += got;
		if (got < CH) break;
	}
	MAB_CUDA(cudaStreamSynchronize(st));
	gzclose(fp);
	for (int i = 0; i < 2; ++i) { MAB_CUDA(cudaFreeHost(pin[i])); MAB_CUDA(cudaEventDestroy(ev[i])); }
	MAB_CUDA(cudaStreamDestroy(st));
	return 0;
}

static void reads_drop(mab_ctx *c)
{
	if (c->rl.started && !c->rl.joined) pthread_join(c->rl.tid, 0);
	if (c->rl.d_text) cudaFree(c->rl.d_text);
	c->rl = mab_ctx::ReadsLoad();
}

/* Start streaming the reads file (FASTA/FASTQ, plain or gzip, "-" = stdin) into HBM in the background; call it before
 * mab_ingest so that the copy hides behind the graph stages.  Optional: mab_write_gfa_reads loads the file itself otherwise. */
int mab_reads_prefetch(mab_ctx_t *c, const char *fn)
{
	reads_drop(c);
	c->rl.fn = fn, c->rl.device = c->dev.device;
	if (pthread_create(&c->rl.tid, 0, reads_loader, &c->rl) != 0) return -1;
	c->rl.started = true;
	return 0;
}

/* ma_ug_seq + ma_ug_print (asm.c:236-290, 77-116): the GFA with unitig sequences, formatted and filled on the GPU.  Returns the
 * bytes written; -1 before mab_unitigs; -2 when the reads file is not in a layout the parallel parser proves (nothing is
 * written: the caller falls back to mab_export_* + ma_ug_seq + ma_ug_print).  A file that cannot be opened gives the GFA
 * without sequences, as the reference does (main.c:193 ignores the return value). */
long mab_write_gfa_reads(mab_ctx_t *c, FILE *fp, const char *fn_reads)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	if (!c->have_ug) return -1;
	MabDev &d = c->dev;
	if (!c->rl.started || c->rl.fn != fn_reads) mab_reads_prefetch(c, fn_reads);
	if (!c->rl.joined) { pthread_join(c->rl.tid, 0); c->rl.joined = true; }
	if (c->rl.rc < 0) { reads_drop(c); return mab_write_gfa(c, fp); }
	DReadsIndex ix;
	const int rc = dg_reads_index(d, c->rl.d_text, c->rl.len, ix);
	if (rc == UGSEQ_UNSUPPORTED) { dg_reads_free(d, ix); reads_drop(c); return -2; }
	if (!c->ug.g.has_idx) dg_arc_index(d, c->ug.g);
	uint64_t *seq_pos = mab_alloc<uint64_t>(d, c->ug.n_utg);
	uint32_t *ioff = nullptr;
	char *d_txt = nullptr;
	const char *ntext = c->name_text ? c->name_text : c->d_text;
	const size_t n = dg_gfa_text(d, c->ug, c->orig_id, c->names.off, c->names.nlen, ntext, c->sub, &d_txt, seq_pos, &ioff);
	if (n) {
		const int gr = dg_ugseq_fill(d, c->rl.d_text, c->rl.len, ix, c->ug, ioff, c->n_seq, c->orig_id, c->names.off, c->names.nlen, ntext, c->sub, seq_pos, d_txt);
		if (gr == UGSEQ_SHORT_RECORD) { // asm.c:263 asserts it
			fprintf(stderr, "[E::ma_ug_seq] a record of '%s' is shorter than the interval the layout keeps of it: wrong reads file?\n", fn_reads);
			abort();
		}
		if (n > c->h_gfa_cap) {
			if (c->h_gfa) MAB_CUDA(cudaFreeHost(c->h_gfa));
			c->h_gfa_cap = n + (n >> 2) + (1 << 20);
			MAB_CUDA(cudaHostAlloc((void**)&c->h_gfa, c->h_gfa_cap, cudaHostAllocDefault));
		}
		MAB_CUDA(cudaMemcpyAsync(c->h_gfa, d_txt, n, cudaMemcpyDeviceToHost, d.stream));
		d.sync();
		if (fwrite(c->h_gfa, 1, n, fp) != n) { fprintf(stderr, "[E::miniasm_b200] short write of the GFA text\n"); exit(74); }
	}
	d.free(d_txt); d.free(ioff); d.free(seq_pos);
	dg_reads_free(d, ix);
	d.sync();
	reads_drop(c);
	return (long)n;
}

/* device-time probe used by bench.py: milliseconds between two points on the context's stream */
void *mab_event_create(void) { cudaEvent_t e; MAB_CUDA(cudaEventCreate(&e)); return e; }
void mab_event_record(mab_ctx_t *c, void *e) { MAB_CUDA(cudaEventRecord((cudaEvent_t)e, c->dev.stream)); }
float mab_event_elapsed_ms(void *a, void *b) { float ms = 0; MAB_CUDA(cudaEventSynchronize((cudaEvent_t)b)); MAB_CUDA(cudaEventElapsedTime(&ms, (cudaEvent_t)a, (cudaEvent_t)b)); return ms; }
void mab_event_destroy(void *e) { MAB_CUDA(cudaEventDestroy((cudaEvent_t)e)); }
void mab_sync(mab_ctx_t *c) { c->dev.sync(); }


/* ------------------------------------------------------------------------------------------------------------
 * Hash-sharded multi-GPU run (SURVEY.md 8e): one process per GPU, read r owned by rank r mod world.
 *   mab_nccl_unique_id (rank 0) -> bytes broadcast by the launcher -> mab_shard_init (all ranks)
 *   mab_load_paf_text/file with THIS RANK'S byte range of the PAF (ranges in rank order, cut at line ends)
 *   mab_ingest_sharded -> mab_select_sharded -> mab_layout_sharded: afterwards every rank holds the same reduced
 *   graph as a single-GPU run of the concatenated PAF would, and mab_unitigs / mab_export_* work as usual.
 * Exchanges: all-gather of distinct names, all-to-all of hits, all-reduce of the interval tables and of the
 * containment / deletion flags, all-gather of raw arcs (for neighbour slabs) and of the reduced arcs.
 * ------------------------------------------------------------------------------------------------------------ */
int mab_nccl_unique_id(void *out128)
{
	ncclUniqueId id;
	MAB_NCCL(ncclGetUniqueId(&id));
	memcpy(out128, &id, sizeof(id) < 128 ? sizeof(id) : 128);
	return (int)sizeof(id);
}

int mab_shard_init(mab_ctx_t *c, int rank, int world, const void *id128)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	c->sc.rank = rank, c->sc.world = world;
	if (world > 1) {
		ncclUniqueId id;
		memcpy(&id, id128, sizeof(id) < 128 ? sizeof(id) : 128);
		MAB_NCCL(ncclCommInitRank(&c->sc.comm, world, id, rank));
	}
	return 0;
}

int mab_ingest_sharded(mab_ctx_t *c, int min_span, int min_match, int bi_dir)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	PhaseTimer pt(d, &c->stats.ms_ingest, "mab_ingest_sharded");
	ctx_reset_reads(c);
	ingest_paf_sharded(d, c->sc, c->d_text, c->text_len, min_span, min_match, bi_dir, c->hits, c->names, &c->name_text, c->ist);
	c->n_seq = c->names.n_seq;
	c->stats.n_lines = c->ist.n_parsed, c->stats.n_hits_stored = c->ist.n_hits, c->stats.n_seq_in = c->ist.n_seq, c->stats.n_name_regrow = c->ist.name_regrow;
	if (!mab_mute && ma_verbose >= 3 && c->sc.rank == 0)
		fprintf(stderr, "[M::%s::%s] read %ld hits; stored %ld hits and %d sequences (%ld bp)\n", "ma_hit_read", sys_timestamp(),
				(long)c->ist.n_parsed, (long)c->ist.n_hits, (int)c->ist.n_seq, (long)c->ist.tot_len);
	return 0;
}

/* mab_load_paf_text + mab_ingest_sharded in one call: this rank's bytes cross PCIe in chunks while the arrived ones are parsed */
int mab_load_ingest_text_sharded(mab_ctx_t *c, const char *text, size_t len, int min_span, int min_match, int bi_dir)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	ctx_reset_reads(c);
	text_reserve(c, len);
	c->text_len = len;
	PhaseTimer pt(d, &c->stats.ms_ingest, "mab_load_ingest_text_sharded");
	ingest_paf_sharded(d, c->sc, c->d_text, c->text_len, min_span, min_match, bi_dir, c->hits, c->names, &c->name_text, c->ist, text);
	c->n_seq = c->names.n_seq;
	c->stats.n_lines = c->ist.n_parsed, c->stats.n_hits_stored = c->ist.n_hits, c->stats.n_seq_in = c->ist.n_seq, c->stats.n_name_regrow = c->ist.name_regrow;
	if (!mab_mute && ma_verbose >= 3 && c->sc.rank == 0)
		fprintf(stderr, "[M::%s::%s] read %ld hits; stored %ld hits and %d sequences (%ld bp)\n", "ma_hit_read", sys_timestamp(),
				(long)c->ist.n_parsed, (long)c->ist.n_hits, (int)c->ist.n_seq, (long)c->ist.tot_len);
	return 0;
}

static void sum_over_ranks(void *ctx, unsigned long long *v, int n) // MabCountHook: the counts of a log line, summed over the ranks
{
	mab_ctx *c = (mab_ctx*)ctx;
	if (!c->sc.active() || n <= 0 || n > 8) return;
	MabDev &d = c->dev;
	unsigned long long *buf = (unsigned long long*)mab_alloc<uint64_t>(d, 8);
	MAB_CUDA(cudaMemcpyAsync(buf, v, 8 * (size_t)n, cudaMemcpyHostToDevice, d.stream));
	MAB_NCCL(ncclAllReduce(buf, buf, (size_t)n, ncclUint64, ncclSum, c->sc.comm, d.stream));
	MAB_CUDA(cudaMemcpyAsync(v, buf, 8 * (size_t)n, cudaMemcpyDeviceToHost, d.stream));
	d.sync();
	d.free(buf);
}

/* default read selection (main.c:119-142 with no -1/-2/-S): dh_select on this rank's hits, with the per-rank interval tables
 * and containment flags completed by all-reduce between its passes */
int mab_select_sharded(mab_ctx_t *c, const ma_opt_t *opt)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	ShardComm &sc = c->sc;
	PhaseTimer pt(d, &c->stats.ms_select, "mab_select_sharded");
	ctx_drop_graphs(c);
	dh_hits_dense(d, c->hits);
	const int msave = mab_mute;
	if (sc.rank != 0) mab_mute = 1; // only rank 0 talks (thread-local: ranks may be threads of one process); the counts it prints are summed over the ranks
	mab_count_hook = sum_over_ranks, mab_count_hook_ctx = c;
	const uint32_t n = c->n_seq;
	SelectHooks hk;
	hk.sub_done = [&](DSub *s) { sc_allreduce(d, sc, s, n, ncclUint64, ncclSum); }; // a row is written by the rank owning the read only
	hk.flags_done = [&](DSub *sub, uint8_t *used, uint32_t n_seq) {
		// containment flags are the top bit of the first word: an element-wise max over ranks is their OR (the other bits agree)
		sc_allreduce(d, sc, sub, (size_t)n_seq * 2, ncclUint32, ncclMax);
		sc_allreduce(d, sc, used, n_seq, ncclUint8, ncclMax);
	};
	select_default(c, opt, hk);
	mab_mute = msave;
	mab_count_hook = nullptr, mab_count_hook_ctx = nullptr;
	c->stats.n_hits_final = c->hits.n, c->stats.n_seq_final = c->n_seq;
	d.sync();
	return 0;
}

__global__ void k_not_flag(const uint8_t *flag, uint32_t n, uint8_t *out)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = !flag[i];
}

/* ma_sg_gen + asg_arc_del_trans sharded, then the cleaning passes on the replicated reduced graph */
int mab_layout_sharded(mab_ctx_t *c, const ma_opt_t *opt)
{
	MAB_CUDA(cudaSetDevice(c->dev.device));
	MabDev &d = c->dev;
	ShardComm &sc = c->sc;
	const int G = sc.world;
	PhaseTimer pt(d, &c->stats.ms_layout, "mab_layout_sharded");
	ctx_drop_graphs(c);
	const int msave = mab_mute;
	if (sc.rank != 0) mab_mute = 1;
	const uint32_t n = c->n_seq;
	uint32_t *len = mab_alloc<uint32_t>(d, n);
	uint8_t *del = mab_alloc<uint8_t>(d, n);
	if (n) MAB_LAUNCH(d, k_sg_len, mab_grid(n, 256), 256, 0, n, c->sub, c->names.slen, c->orig_id, len, del);
	HitArcParams p = { opt->max_hang, opt->int_frac, opt->min_ovlp };
	c->hits.n_seq = n;
	DGraph loc;                                             // arcs of the reads this rank owns, sorted
	dh_sg_emit(d, c->hits, len, del, p, loc);
	d.free(len); d.free(del);
	sc_allreduce(d, sc, loc.seq, n, ncclUint32, ncclMax);   // deletion flags raised by any rank (top bit; lengths agree)
	dg_arc_rm(d, loc, nullptr);
	DGraph &g = c->sg;
	uint32_t n_keep = 0;
	DArc *keep = nullptr;
	uint64_t n_red_all = 0, tot = 0;
	std::vector<uint64_t> cnt = sc_allgather_u64(d, sc, loc.n_arc);
	for (int r = 0; r < G; ++r) tot += cnt[r];
	if (tot >= (1ull << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 arcs in the graph\n"); exit(73); }
	c->stats.n_arc_sg = tot;
	if (MAB_V(1)) fprintf(stderr, "[M::%s] read %d arcs\n", "ma_sg_gen", (int)tot);
	// ---- neighbour slabs: peer access over NVLink when every rank can offer it (shard_comm.cuh), else an all-gather of all arcs
	std::vector<void*> peer_any;
	const bool p2p = sc_peer_ptrs(d, sc, loc.arc, peer_any);
	std::vector<const DArc*> peer_ptr((size_t)G, nullptr);
	for (int r = 0; r < G; ++r) peer_ptr[r] = (const DArc*)peer_any[r];
	if (p2p) {
		if (!loc.has_idx) dg_arc_index(d, loc);                 // slabs of the vertices this rank owns
		uint64_t *nidx = mab_alloc<uint64_t>(d, (size_t)n * 2);
		if (n) MAB_CUDA(cudaMemcpyAsync(nidx, loc.idx, (size_t)n * 16, cudaMemcpyDeviceToDevice, d.stream));
		sc_allreduce(d, sc, nidx, (size_t)n * 2, ncclUint64, ncclSum); // every vertex is indexed by exactly one rank
		const DArc **d_peer = (const DArc**)d.alloc(sizeof(void*) * (size_t)G);
		MAB_CUDA(cudaMemcpyAsync(d_peer, peer_ptr.data(), sizeof(void*) * (size_t)G, cudaMemcpyHostToDevice, d.stream));
		uint8_t *flag = nullptr;
		uint32_t n_red = dg_del_trans_flags(d, loc, (uint32_t)opt->gap_fuzz, 0, 0xffffffffu, &flag, d_peer, nidx, c->orig_id, (uint32_t)G);
		c->stats.ms_del_trans_kernel = g_del_trans_stats.kernel_ms, c->stats.trans_inner = g_del_trans_stats.inner_iters;
		std::vector<uint64_t> reds = sc_allgather_u64(d, sc, n_red);
		for (int r = 0; r < G; ++r) n_red_all += reds[r];
		keep = mab_alloc<DArc>(d, loc.n_arc);
		if (loc.n_arc) {
			uint8_t *nf = mab_alloc<uint8_t>(d, loc.n_arc);
			MAB_LAUNCH(d, k_not_flag, mab_grid(loc.n_arc, 256), 256, 0, flag, loc.n_arc, nf);
			size_t tb = 0;
			unsigned long long *d_n = d.d_scal + SC_NSEL;
			cub::DeviceSelect::Flagged(nullptr, tb, loc.arc, nf, keep, d_n, (int)loc.n_arc, d.stream);
			void *tmp = d.tmp(tb);
			cub::DeviceSelect::Flagged(tmp, tb, loc.arc, nf, keep, d_n, (int)loc.n_arc, d.stream);
			++d.n_lib;
			n_keep = (uint32_t)d.get_scal(SC_NSEL);
			d.free(nf);
		}
		d.free(flag); d.free(nidx); d.free((void*)d_peer);
		dg_set_nseq(d, g, n);
		if (n) MAB_CUDA(cudaMemcpyAsync(g.seq, loc.seq, (size_t)n * 4, cudaMemcpyDeviceToDevice, d.stream));
		g.len_bits = loc.len_bits, g.is_symm = false;
		c->have_sg = true;
		c->stats.n_arc_trans_in = loc.n_arc;
	} else {
	// all ranks' raw arcs, concatenated in rank order: every vertex's slab is contiguous in it, which is all the index needs
	uint64_t my_off = 0, run = 0;
	std::vector<uint64_t> bytes(G);
	for (int r = 0; r < G; ++r) { if (r == sc.rank) my_off = run; run += cnt[r]; bytes[r] = cnt[r] * sizeof(DArc); }
	dg_set_nseq(d, g, n);
	dg_reserve(d, g, tot ? tot : 1);
	if (n) MAB_CUDA(cudaMemcpyAsync(g.seq, loc.seq, (size_t)n * 4, cudaMemcpyDeviceToDevice, d.stream));
	sc_allgather_v(d, sc, loc.arc, bytes, g.arc);
	g.n_arc = (uint32_t)tot, g.is_srt = true, g.is_symm = false, g.len_bits = loc.len_bits;
	dg_arc_index(d, g);
	c->have_sg = true;
	// transitive reduction of the vertices this rank owns (their slabs start inside its block of the concatenation)
	uint8_t *flag = nullptr;
	uint32_t n_red = dg_del_trans_flags(d, g, (uint32_t)opt->gap_fuzz, (uint32_t)my_off, (uint32_t)(my_off + cnt[sc.rank]), &flag);
	c->stats.ms_del_trans_kernel = g_del_trans_stats.kernel_ms, c->stats.trans_inner = g_del_trans_stats.inner_iters;
	std::vector<uint64_t> reds = sc_allgather_u64(d, sc, n_red);
	for (int r = 0; r < G; ++r) n_red_all += reds[r];
	c->stats.n_arc_trans_in = cnt[sc.rank]; // arcs of the vertices this rank reduces
	// survivors of the own block
	keep = mab_alloc<DArc>(d, cnt[sc.rank]);
	if (cnt[sc.rank]) {
		uint8_t *nf = mab_alloc<uint8_t>(d, cnt[sc.rank]);
		MAB_LAUNCH(d, k_not_flag, mab_grid(cnt[sc.rank], 256), 256, 0, flag + my_off, (uint32_t)cnt[sc.rank], nf);
		size_t tb = 0;
		unsigned long long *d_n = d.d_scal + SC_NSEL;
		cub::DeviceSelect::Flagged(nullptr, tb, g.arc + my_off, nf, keep, d_n, (int)cnt[sc.rank], d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceSelect::Flagged(tmp, tb, g.arc + my_off, nf, keep, d_n, (int)cnt[sc.rank], d.stream);
		++d.n_lib;
		n_keep = (uint32_t)d.get_scal(SC_NSEL);
		d.free(nf);
	}
	d.free(flag);
	}
	c->stats.n_reduced = n_red_all;
	if (MAB_V(1)) fprintf(stderr, "[M::%s] transitively reduced %d arcs\n", "asg_arc_del_trans", (int)n_red_all);
	// survivors -> all ranks; their stable sort by (vertex, length) is the single-GPU arc array
	std::vector<uint64_t> bytes(G);
	std::vector<uint64_t> kc = sc_allgather_u64(d, sc, n_keep);
	uint64_t ktot = 0;
	for (int r = 0; r < G; ++r) { ktot += kc[r]; bytes[r] = kc[r] * sizeof(DArc); }
	DArc *all = mab_alloc<DArc>(d, ktot);
	sc_allgather_v(d, sc, keep, bytes, all);
	d.free(keep);
	dg_reserve(d, g, ktot ? ktot : 1);
	if (ktot) MAB_CUDA(cudaMemcpyAsync(g.arc, all, ktot * sizeof(DArc), cudaMemcpyDeviceToDevice, d.stream));
	d.free(all);
	g.n_arc = (uint32_t)ktot, g.is_srt = false, g.has_idx = false;
	dg_cleanup(d, g);                                       // stable radix sort by ul + index (nothing left to remove)
	if (n_red_all) dg_symm(d, g);                           // asg.c:188-191
	dg_free(d, loc);
	layout_tail(c, opt, 100);
	mab_mute = msave;
	return 0;
}
}
