// gunzip_dev.cu -- the kernels of the GPU gzip decoder (gunzip_dev.cuh, DESIGN.md section 3c) over the inflate.cuh core:
//   k_gz_find     one block per chunk of compressed bytes: the first bit offset that passes the block-start test
//   k_gz_compact  unit starts = the true start (bit 0) + the chunks' guesses, ascending
//   k_gz_decode   pass 1, one thread per unit: decode with unknown history into a 32 KiB ring of bytes and window markers
//   k_gz_chain    walk the units from the true start along the confirmed landings; output offsets and member slots
//   k_gz_window   in chain order, the resolved 32 KiB window after each chained unit
//   k_gz_resolve  pass 2, one thread per chained unit: decode again with the true window, bytes straight into place
//   k_gz_crc_seg / k_gz_crc_member   raw CRC-32 per fixed segment, joined per member by GF(2) shifts, checked with ISIZE
// and GzStream, which runs the same kernels over one compressed segment at a time (k_gz_chain_seg, gzstream.cuh).
#include "gunzip_dev.cuh"
#include "inflate.cuh"
#include "gzstream.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <vector>

#define GZ_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
	fprintf(stderr, "[E::miniasm_b200] %s failed at %s:%d: %s\n", #x, __FILE__, __LINE__, cudaGetErrorString(e_)); \
	exit(70); } } while (0)

static const size_t GZ_CHUNK = 64u << 10;   // compressed bytes per chunk (DESIGN.md 3c: measured on config 3)
static const size_t GZ_SEG = 16u << 10;     // output bytes per CRC segment
static const int GZ_TRIAL = 256;            // symbols of the block-start test's trial decode
static const uint64_t GZ_NONE = ~0ull;

static double sys_wall_ms() { timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e3 + t.tv_nsec * 1e-6; }

// device scalars
enum { GS_NU = 0, GS_NC, GS_TOTAL, GS_MEMBERS, GS_ERR, GS_CONF, GS_KIND, GS_NEXT, GS_OLEN0, GS_N };

__global__ void __launch_bounds__(256) k_gz_find(const uint8_t *gz, uint64_t n, uint64_t chunk, uint64_t *guess)
{
	__shared__ unsigned long long found;
	const uint64_t i = blockIdx.x + 1, b0 = i * chunk * 8, b1 = (i + 1) * chunk < n ? (i + 1) * chunk * 8 : n * 8;
	if (threadIdx.x == 0) found = GZ_NONE;
	__syncthreads();
	InfTables t;
	for (uint64_t base = b0; base < b1; base += blockDim.x) {
		const uint64_t b = base + threadIdx.x;
		if (b < b1 && inf_guess_test(gz, n, b, t, GZ_TRIAL)) atomicMin(&found, (unsigned long long)b);
		__syncthreads();
		if (found != GZ_NONE) break;
	}
	if (threadIdx.x == 0) guess[i] = found;
}

__global__ void k_gz_compact(const uint64_t *guess, uint64_t n_chunks, uint64_t *starts, unsigned long long *sc, uint64_t first = 0)
{
	uint64_t k = 0;
	starts[k++] = first;
	for (uint64_t i = 1; i < n_chunks; ++i) if (guess[i] != GZ_NONE) starts[k++] = guess[i];
	sc[GS_NU] = k;
}

__global__ void __launch_bounds__(32) k_gz_decode(const uint8_t *gz, uint64_t n, const uint64_t *starts, uint32_t nu, uint16_t *ring,
                                                  int *st, uint32_t *land, uint64_t *olen, int64_t *mat, uint32_t *nmem, bool hdr0 = true)
{
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= nu) return;
	InfTables t;
	InfOutMark o;
	o.begin(ring + (size_t)u * INF_WIN);
	uint32_t j = u + 1;
	st[u] = inf_run(gz, n, starts[u], u == 0 && hdr0, starts, nu, &j, t, o);
	land[u] = j, olen[u] = o.p, mat[u] = o.member_at, nmem[u] = o.n_members;
}

__global__ void k_gz_chain(const int *st, const uint32_t *land, const uint64_t *olen, const uint32_t *nmem, uint32_t nu,
                           uint32_t *chain, uint64_t *off, uint32_t *mbase, unsigned long long *sc)
{
	uint64_t total = 0, members = 0, c = 0;
	for (uint32_t u = 0;; ++c) {
		if (st[u] < 0) { sc[GS_ERR] = 1; return; }
		chain[c] = u, off[c] = total, mbase[c] = (uint32_t)members;
		total += olen[u], members += nmem[u];
		if (st[u] == INF_END) break;
		u = land[u]; // > u: the chain always moves on
	}
	sc[GS_NC] = c + 1, sc[GS_TOTAL] = total, sc[GS_MEMBERS] = members, sc[GS_CONF] = c;
}

__global__ void __launch_bounds__(1024) k_gz_window(const uint32_t *chain, uint32_t nc, const uint16_t *ring, const uint64_t *olen,
                                                    const int64_t *mat, uint8_t *win, uint32_t *valid)
{
	for (uint32_t c = 0; c < nc; ++c) {
		const uint32_t u = chain[c];
		const uint8_t *wi = win + (size_t)c * INF_WIN;
		uint8_t *wo = win + (size_t)(c + 1) * INF_WIN;
		for (uint32_t k = threadIdx.x; k < INF_WIN; k += blockDim.x) wo[k] = inf_window_byte(ring + (size_t)u * INF_WIN, olen[u], wi, k);
		if (threadIdx.x == 0) valid[c + 1] = inf_window_valid(valid[c], olen[u], mat[u]);
		__syncthreads();
	}
}

__global__ void __launch_bounds__(32) k_gz_resolve(const uint8_t *gz, uint64_t n, const uint64_t *starts, uint32_t nu, const uint32_t *chain,
                                                   uint32_t nc, const uint64_t *off, const uint32_t *mbase, const int *st, const uint32_t *land,
                                                   const uint64_t *olen, const uint32_t *nmem, const uint8_t *win, const uint32_t *valid,
                                                   uint8_t *out, uint64_t *m_end, uint32_t *m_crc, uint32_t *m_isize, unsigned long long *sc,
                                                   bool hdr0 = true)
{
	const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= nc) return;
	const uint32_t u = chain[c];
	InfTables t;
	InfOutByte o;
	o.out = out + off[c], o.win = win + (size_t)c * INF_WIN, o.p = 0, o.cap = olen[u], o.lim = -(int64_t)valid[c];
	o.m_end = m_end + mbase[c], o.m_crc = m_crc + mbase[c], o.m_isize = m_isize + mbase[c], o.n_members = 0, o.m_cap = nmem[u];
	uint32_t j = u + 1;
	const int r = inf_run(gz, n, starts[u], u == 0 && hdr0, starts, nu, &j, t, o);
	if (r != st[u] || o.p != olen[u] || o.n_members != nmem[u] || (r == INF_LAND && j != land[u])) { sc[GS_ERR] = 1; return; }
	for (uint32_t k = 0; k < o.n_members; ++k) o.m_end[k] += off[c];
}

__global__ void k_gz_crc_seg(const uint8_t *txt, uint64_t total, uint64_t seg, uint32_t *sc)
{
	__shared__ uint32_t tab[256];
	if (threadIdx.x < 256) {
		uint32_t c = threadIdx.x;
		for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (c & 1 ? INF_CRC_POLY : 0);
		tab[threadIdx.x] = c;
	}
	__syncthreads();
	const uint64_t n_seg = (total + seg - 1) / seg;
	for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < n_seg; s += (uint64_t)gridDim.x * blockDim.x) {
		const uint64_t a = s * seg, l = total - a < seg ? total - a : seg;
		const uint32_t *w = (const uint32_t*)(txt + a);
		uint32_t c = 0;
		uint64_t i = 0;
		if (((uintptr_t)txt & 3) == 0) for (; i + 4 <= l; i += 4) { // segments start at multiples of 16 KiB
			const uint32_t v = w[i >> 2];
			c = tab[(c ^ v) & 255] ^ (c >> 8);
			c = tab[(c ^ (v >> 8)) & 255] ^ (c >> 8);
			c = tab[(c ^ (v >> 16)) & 255] ^ (c >> 8);
			c = tab[(c ^ (v >> 24)) & 255] ^ (c >> 8);
		}
		for (; i < l; ++i) c = tab[(c ^ txt[a + i]) & 255] ^ (c >> 8);
		sc[s] = c;
	}
}

// one block per member [a, b): its head piece up to the first segment boundary, the whole segments, its tail piece; each
// thread joins a contiguous run of them, then the block joins the runs in order.  carry != nullptr (GzStream): block 0 continues
// the member open before the text (raw CRC carry[0] over carry[1] bytes), and block n_members, the piece [m_end[n-1], total)
// of the member left open, writes its joined raw CRC and length to carry_out
__global__ void __launch_bounds__(128) k_gz_crc_member(const uint8_t *txt, uint64_t seg, const uint32_t *seg_crc, const uint64_t *m_end,
                                                       const uint32_t *m_crc, const uint32_t *m_isize, unsigned long long *sc,
                                                       uint32_t n_members = ~0u, uint64_t total = 0,
                                                       const unsigned long long *carry = nullptr, unsigned long long *carry_out = nullptr)
{
	__shared__ uint32_t tab[256], x2k[64], r_crc[128];
	__shared__ uint64_t r_len[128];
	const uint32_t m = blockIdx.x, tid = threadIdx.x;
	for (uint32_t e = tid; e < 256; e += blockDim.x) {
		uint32_t c = e;
		for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (c & 1 ? INF_CRC_POLY : 0);
		tab[e] = c;
	}
	if (tid == 0) inf_x2k_table(x2k);
	__syncthreads();
	const uint64_t a = m ? m_end[m - 1] : 0, b = m < n_members ? m_end[m] : total;
	uint64_t A = (a + seg - 1) / seg * seg, B = b / seg * seg;
	if (A > b) A = b;
	if (B < A) B = A;
	const uint64_t n_full = (B - A) / seg, n_items = n_full + 2; // head, full segments, tail
	const uint64_t per = (n_items + blockDim.x - 1) / blockDim.x;
	const uint32_t xs = inf_x8n(x2k, seg);
	uint32_t raw = 0;
	uint64_t len = 0;
	for (uint64_t it = tid * per; it < n_items && it < (tid + 1) * per; ++it) {
		if (it == 0) raw = inf_crc_raw(tab, 0, txt + a, A - a), len = A - a;
		else if (it <= n_full) raw = inf_gf2_mul(raw, xs) ^ seg_crc[A / seg + it - 1], len += seg;
		else raw = inf_crc_join(x2k, raw, inf_crc_raw(tab, 0, txt + B, b - B), b - B), len += b - B;
	}
	r_crc[tid] = raw, r_len[tid] = len;
	__syncthreads();
	for (uint32_t s = 1; s < blockDim.x; s <<= 1) {
		if (tid % (2 * s) == 0 && tid + s < blockDim.x) {
			r_crc[tid] = inf_crc_join(x2k, r_crc[tid], r_crc[tid + s], r_len[tid + s]);
			r_len[tid] += r_len[tid + s];
		}
		__syncthreads();
	}
	if (tid == 0 && !carry && (inf_crc_final(x2k, r_crc[0], b - a) != m_crc[m] || (uint32_t)(b - a) != m_isize[m])) sc[GS_ERR] = 1;
	if (tid == 0 && carry) {
		uint32_t raw = r_crc[0];
		uint64_t l = b - a;
		gzs_piece(x2k, (uint32_t)carry[0], carry[1], m, raw, l);
		if (m == n_members) carry_out[0] = raw, carry_out[1] = l;
		else if (!gzs_member_ok(x2k, raw, l, m_crc[m], m_isize[m])) sc[GS_ERR] = 1;
	}
}

// the chain of one segment of a stream (gzs_chain); the next segment's start bit and unit 0's output length for the host
__global__ void k_gz_chain_seg(const int *st, const uint32_t *land, const uint64_t *olen, const uint32_t *nmem, const uint64_t *starts, bool final,
                               uint64_t cap, uint32_t *chain, uint64_t *off, uint32_t *mbase, unsigned long long *sc)
{
	GzsChain r;
	gzs_chain(st, land, olen, nmem, final, cap, chain, off, mbase, r);
	sc[GS_NC] = r.nc, sc[GS_TOTAL] = r.total, sc[GS_MEMBERS] = r.members, sc[GS_KIND] = r.kind;
	sc[GS_NEXT] = starts[r.stop], sc[GS_CONF] = r.nc ? r.nc - 1 : 0;
	sc[GS_OLEN0] = r.nc == 0 ? olen[0] : r.kind == GZS_STOP && st[r.stop] == INF_LAND ? olen[r.stop] : 0; // (the unit that did not fit)
}

namespace {
struct Scratch { // every allocation of one inflate, freed together; tracks the peak
	GzMem &mem;
	std::vector<std::pair<void*, size_t>> live;
	size_t now = 0, peak = 0;
	explicit Scratch(GzMem &m) : mem(m) {}
	template <typename T> T *get(size_t n)
	{
		const size_t bytes = (n ? n : 1) * sizeof(T);
		void *p = mem.alloc(bytes);
		live.push_back({p, bytes});
		now += bytes, peak = now > peak ? now : peak;
		return (T*)p;
	}
	void put(void *p)
	{
		for (size_t i = 0; i < live.size(); ++i) if (live[i].first == p) { now -= live[i].second; live.erase(live.begin() + i); break; }
		mem.free(p);
	}
	~Scratch() { for (auto &e : live) mem.free(e.first); }
};
}

int gz_inflate_dev(cudaStream_t st, GzMem &mem, const uint8_t *gz, size_t len, char *(*out)(void *ctx, size_t n), void *ctx,
                   size_t *out_len, GzStats *stats, size_t chunk)
{
	*out_len = 0;
	if (len < 18) return GZ_REJECT; // shorter than a header and a trailer
	if (!chunk) chunk = GZ_CHUNK;
	Scratch s(mem);
	cudaEvent_t ev[7];
	for (int i = 0; i < 7; ++i) GZ_CUDA(cudaEventCreate(&ev[i]));
	unsigned long long *d_sc = s.get<unsigned long long>(GS_N), h_sc[GS_N];
	GZ_CUDA(cudaMemsetAsync(d_sc, 0, GS_N * sizeof(unsigned long long), st));
	auto fetch = [&]() {
		GZ_CUDA(cudaMemcpyAsync(h_sc, d_sc, sizeof(h_sc), cudaMemcpyDeviceToHost, st));
		GZ_CUDA(cudaStreamSynchronize(st));
	};
	int rc = GZ_REJECT;
	const uint64_t n_chunks = (len + chunk - 1) / chunk;
	GZ_CUDA(cudaEventRecord(ev[0], st));
	// find + compact
	uint64_t *guess = s.get<uint64_t>(n_chunks), *starts = s.get<uint64_t>(n_chunks);
	if (n_chunks > 1) { k_gz_find<<<(unsigned)(n_chunks - 1), 256, 0, st>>>(gz, len, chunk, guess); GZ_CUDA(cudaGetLastError()); }
	k_gz_compact<<<1, 1, 0, st>>>(guess, n_chunks, starts, d_sc);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev[1], st));
	fetch();
	const uint32_t nu = (uint32_t)h_sc[GS_NU];
	s.put(guess);
	// pass 1
	uint16_t *ring = s.get<uint16_t>((size_t)nu * INF_WIN);
	int *ust = s.get<int>(nu);
	uint32_t *land = s.get<uint32_t>(nu), *nmem = s.get<uint32_t>(nu);
	uint64_t *olen = s.get<uint64_t>(nu);
	int64_t *mat = s.get<int64_t>(nu);
	k_gz_decode<<<(nu + 31) / 32, 32, 0, st>>>(gz, len, starts, nu, ring, ust, land, olen, mat, nmem);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev[2], st));
	// chain
	uint32_t *chain = s.get<uint32_t>(nu), *mbase = s.get<uint32_t>(nu);
	uint64_t *off = s.get<uint64_t>(nu);
	k_gz_chain<<<1, 1, 0, st>>>(ust, land, olen, nmem, nu, chain, off, mbase, d_sc);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev[3], st));
	fetch();
	const uint32_t nc = (uint32_t)h_sc[GS_NC];
	const uint64_t total = h_sc[GS_TOTAL], members = h_sc[GS_MEMBERS];
	float ms[6] = { 0, 0, 0, 0, 0, 0 };
	if (!h_sc[GS_ERR]) {
		// window
		uint8_t *win = s.get<uint8_t>((size_t)(nc + 1) * INF_WIN);
		uint32_t *valid = s.get<uint32_t>(nc + 1);
		GZ_CUDA(cudaMemsetAsync(win, 0, INF_WIN, st));
		GZ_CUDA(cudaMemsetAsync(valid, 0, sizeof(uint32_t), st));
		k_gz_window<<<1, 1024, 0, st>>>(chain, nc, ring, olen, mat, win, valid);
		GZ_CUDA(cudaGetLastError());
		GZ_CUDA(cudaEventRecord(ev[4], st));
		// resolve
		char *dst = out(ctx, total);
		uint64_t *m_end = s.get<uint64_t>(members);
		uint32_t *m_crc = s.get<uint32_t>(members), *m_isize = s.get<uint32_t>(members);
		k_gz_resolve<<<(nc + 31) / 32, 32, 0, st>>>(gz, len, starts, nu, chain, nc, off, mbase, ust, land, olen, nmem, win, valid,
		                                            (uint8_t*)dst, m_end, m_crc, m_isize, d_sc);
		GZ_CUDA(cudaGetLastError());
		GZ_CUDA(cudaEventRecord(ev[5], st));
		// crc
		const uint64_t n_seg = (total + GZ_SEG - 1) / GZ_SEG;
		uint32_t *seg_crc = s.get<uint32_t>(n_seg);
		if (n_seg) { k_gz_crc_seg<<<(unsigned)((n_seg + 255) / 256), 256, 0, st>>>((const uint8_t*)dst, total, GZ_SEG, seg_crc); GZ_CUDA(cudaGetLastError()); }
		if (members) { k_gz_crc_member<<<(unsigned)members, 128, 0, st>>>((const uint8_t*)dst, GZ_SEG, seg_crc, m_end, m_crc, m_isize, d_sc); GZ_CUDA(cudaGetLastError()); }
		GZ_CUDA(cudaEventRecord(ev[6], st));
		fetch();
		if (!h_sc[GS_ERR]) rc = GZ_OK, *out_len = total;
		for (int i = 0; i < 6; ++i) GZ_CUDA(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
	}
	if (stats) {
		stats->ms_find = ms[0], stats->ms_decode = ms[1], stats->ms_chain = ms[2], stats->ms_window = ms[3], stats->ms_resolve = ms[4], stats->ms_crc = ms[5];
		stats->n_chunks = n_chunks, stats->n_units = nu, stats->n_chain = nc, stats->n_confirmed = h_sc[GS_CONF];
		stats->n_members = members, stats->out_len = rc == GZ_OK ? total : 0, stats->scratch_peak = s.peak;
	}
	for (int i = 0; i < 7; ++i) GZ_CUDA(cudaEventDestroy(ev[i]));
	return rc;
}

// ---- the streaming decoder ---------------------------------------------------------------------------------------------
enum { GZ_GROW = -4 }; // (step only: unit 0 needs a longer segment)

// Pass 1 of one segment, which needs no history: its compressed bytes, the units (found on the device; the ring and the per-unit
// arrays are sized for one unit per chunk, so nothing returns to the host before the decode is queued) and their speculative
// decode, all on one stream.  The next segment's pass 1 runs on a second stream while the current one is resolved and parsed.
struct GzP1 {
	Scratch s;
	uint64_t base = 0, n = 0, bit = 0, chunk = 0, n_chunks = 0;
	bool final = false, hdr = false;
	uint8_t *gz = nullptr;
	uint64_t *starts = nullptr, *olen = nullptr;
	unsigned long long *d_sc = nullptr;
	uint16_t *ring = nullptr;
	int *ust = nullptr;
	uint32_t *land = nullptr, *nmem = nullptr;
	int64_t *mat = nullptr;
	cudaEvent_t ev[3];
	explicit GzP1(GzMem &m) : s(m) { for (int i = 0; i < 3; ++i) GZ_CUDA(cudaEventCreate(&ev[i])); }
	~GzP1() { for (int i = 0; i < 3; ++i) GZ_CUDA(cudaEventDestroy(ev[i])); }
};

// k_gz_decode over the units k_gz_compact listed (their number is read on the device)
__global__ void __launch_bounds__(32) k_gz_decode_n(const uint8_t *gz, uint64_t n, const uint64_t *starts, const unsigned long long *d_nu,
                                                    uint16_t *ring, int *st, uint32_t *land, uint64_t *olen, int64_t *mat, uint32_t *nmem, bool hdr0)
{
	const uint32_t nu = (uint32_t)*d_nu, u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= nu) return;
	InfTables t;
	InfOutMark o;
	o.begin(ring + (size_t)u * INF_WIN);
	uint32_t j = u + 1;
	st[u] = inf_run(gz, n, starts[u], u == 0 && hdr0, starts, nu, &j, t, o);
	land[u] = j, olen[u] = o.p, mat[u] = o.member_at, nmem[u] = o.n_members;
}

GzStream::GzStream(cudaStream_t st, GzMem &mem, GzInput &in, uint64_t len, size_t chunk) : st_(st), mem_(mem), in_(in), len_(len), chunk_(chunk)
{
	memset(&sum, 0, sizeof(sum));
	GZ_CUDA(cudaStreamCreateWithFlags(&st2_, cudaStreamNonBlocking));
	hist_ = (uint8_t*)mem_.alloc(INF_WIN);
	valid_ = (uint32_t*)mem_.alloc(sizeof(uint32_t));
	carry_ = (unsigned long long*)mem_.alloc(4 * sizeof(unsigned long long));
	for (int i = 0; i < 7; ++i) GZ_CUDA(cudaEventCreate(&ev_[i]));
	rewind();
}

GzStream::~GzStream()
{
	drop_prefetch();
	GZ_CUDA(cudaStreamSynchronize(st_));
	mem_.free(hist_), mem_.free(valid_), mem_.free(carry_);
	for (int i = 0; i < 7; ++i) GZ_CUDA(cudaEventDestroy(ev_[i]));
	GZ_CUDA(cudaStreamDestroy(st2_));
}

void GzStream::drop_prefetch()
{
	if (!pre_) return;
	GZ_CUDA(cudaStreamSynchronize(st2_)); // (its scratch goes back to the allocator only once nothing uses it)
	delete pre_;
	pre_ = nullptr;
}

void GzStream::rewind()
{
	drop_prefetch();
	pos_ = 0, need_ = 0, next_seg_ = 0, hdr_ = true, done_ = false; // (the ratio seen so far stays: it sizes the next pass's segments)
	GZ_CUDA(cudaMemsetAsync(hist_, 0, INF_WIN, st_));
	GZ_CUDA(cudaMemsetAsync(valid_, 0, sizeof(uint32_t), st_));
	GZ_CUDA(cudaMemsetAsync(carry_, 0, 4 * sizeof(unsigned long long), st_));
}

// read, find and decode segment [base, base + n) starting at absolute bit `bit`, queued on st; nullptr on a read error
GzP1 *GzStream::p1_launch(uint64_t bit, uint64_t n, bool hdr, cudaStream_t st)
{
	GzP1 *p = new GzP1(mem_);
	p->base = bit >> 3, p->bit = bit, p->n = n, p->final = p->base + n == len_, p->hdr = hdr;
	p->gz = p->s.get<uint8_t>(n);
	const double t0 = sys_wall_ms();
	if (!in_.read(p->base, n, p->gz, st)) { GZ_CUDA(cudaStreamSynchronize(st)); delete p; return nullptr; }
	ms_read += sys_wall_ms() - t0;
	p->d_sc = p->s.get<unsigned long long>(GS_N);
	GZ_CUDA(cudaMemsetAsync(p->d_sc, 0, GS_N * sizeof(unsigned long long), st));
	p->chunk = chunk_ ? chunk_ : gzs_chunk_for(n), p->n_chunks = (n + p->chunk - 1) / p->chunk;
	const uint64_t nch = p->n_chunks;
	GZ_CUDA(cudaEventRecord(p->ev[0], st));
	uint64_t *guess = p->s.get<uint64_t>(nch);
	p->starts = p->s.get<uint64_t>(nch);
	if (nch > 1) { k_gz_find<<<(unsigned)(nch - 1), 256, 0, st>>>(p->gz, n, p->chunk, guess); GZ_CUDA(cudaGetLastError()); }
	k_gz_compact<<<1, 1, 0, st>>>(guess, nch, p->starts, p->d_sc, bit & 7);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(p->ev[1], st));
	p->ring = p->s.get<uint16_t>((size_t)nch * INF_WIN);
	p->ust = p->s.get<int>(nch);
	p->land = p->s.get<uint32_t>(nch), p->nmem = p->s.get<uint32_t>(nch);
	p->olen = p->s.get<uint64_t>(nch);
	p->mat = p->s.get<int64_t>(nch);
	k_gz_decode_n<<<(unsigned)((nch + 31) / 32), 32, 0, st>>>(p->gz, n, p->starts, p->d_sc + GS_NU, p->ring, p->ust, p->land, p->olen, p->mat, p->nmem, hdr);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(p->ev[2], st));
	return p;
}

int64_t GzStream::fill(char *dst, size_t cap, size_t *need)
{
	if (len_ < 18) return GZ_REJECT;
	if (!done_ && gzs_room_short(need_, cap)) { if (need) *need = need_; return GZ_SMALL; }
	while (!done_) {
		const uint64_t base = pos_ >> 3;
		uint64_t seg = next_seg_ ? next_seg_ : gzs_seg_len(cap, in_used_, out_made_);
		for (;;) {
			GzP1 *p = nullptr;
			if (pre_ && pre_->bit == pos_ && pre_->n == (seg < len_ - base ? seg : len_ - base)) {
				p = pre_, pre_ = nullptr;
				GZ_CUDA(cudaStreamWaitEvent(st_, p->ev[2], 0)); // its pass 1 is done before the chain reads it
			} else {
				drop_prefetch();
				p = p1_launch(pos_, seg < len_ - base ? seg : len_ - base, hdr_, st_);
				if (!p) return GZ_REJECT;
			}
			const int64_t r = step(*p, (uint8_t*)dst, cap, need);
			const uint64_t n = p->n;
			delete p; // (what the main stream still queues on its scratch runs before any later use of it: one stream)
			if (r == GZ_GROW) { drop_prefetch(); seg = 2 * n, ++n_grown; continue; }
			if (r < 0) drop_prefetch();
			if (r != 0 || done_) return r;
			break; // only empty output taken: on to the next segment
		}
	}
	return 0;
}

int64_t GzStream::step(GzP1 &p, uint8_t *dst, uint64_t cap, size_t *need)
{
	Scratch &s = p.s;
	++n_segments;
	unsigned long long *d_sc = p.d_sc, h_sc[GS_N];
	auto fetch = [&]() {
		GZ_CUDA(cudaMemcpyAsync(h_sc, d_sc, sizeof(h_sc), cudaMemcpyDeviceToHost, st_));
		GZ_CUDA(cudaStreamSynchronize(st_));
	};
	const uint64_t nch = p.n_chunks, n = p.n;
	GZ_CUDA(cudaEventRecord(ev_[0], st_));
	uint32_t *chain = s.get<uint32_t>(nch), *mbase = s.get<uint32_t>(nch);
	uint64_t *off = s.get<uint64_t>(nch);
	k_gz_chain_seg<<<1, 1, 0, st_>>>(p.ust, p.land, p.olen, p.nmem, p.starts, p.final, cap, chain, off, mbase, d_sc);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev_[1], st_));
	fetch();
	float ms[6] = { 0, 0, 0, 0, 0, 0 };
	GZ_CUDA(cudaEventElapsedTime(&ms[0], p.ev[0], p.ev[1]));
	GZ_CUDA(cudaEventElapsedTime(&ms[1], p.ev[1], p.ev[2]));
	GZ_CUDA(cudaEventElapsedTime(&ms[2], ev_[0], ev_[1]));
	const uint32_t nu = (uint32_t)h_sc[GS_NU];
	sum.ms_find += ms[0], sum.ms_decode += ms[1], sum.ms_chain += ms[2];
	sum.n_chunks += nch, sum.n_units += nu;
	const int kind = (int)h_sc[GS_KIND];
	if (kind == GZS_BAD) return GZ_REJECT;
	if (kind == GZS_GROW) return GZ_GROW;
	if (kind == GZS_SMALL) { if (need) *need = h_sc[GS_OLEN0]; return GZ_SMALL; }
	const uint32_t nc = (uint32_t)h_sc[GS_NC];
	const uint64_t total = h_sc[GS_TOTAL], members = h_sc[GS_MEMBERS], next = h_sc[GS_NEXT], need_next = h_sc[GS_OLEN0];
	// windows from the carried history
	uint8_t *win = s.get<uint8_t>((size_t)(nc + 1) * INF_WIN);
	uint32_t *valid = s.get<uint32_t>(nc + 1);
	GZ_CUDA(cudaMemcpyAsync(win, hist_, INF_WIN, cudaMemcpyDeviceToDevice, st_));
	GZ_CUDA(cudaMemcpyAsync(valid, valid_, sizeof(uint32_t), cudaMemcpyDeviceToDevice, st_));
	GZ_CUDA(cudaEventRecord(ev_[2], st_));
	k_gz_window<<<1, 1024, 0, st_>>>(chain, nc, p.ring, p.olen, p.mat, win, valid);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev_[3], st_));
	// where the next segment starts is known now: once the windows are built (the ring is their last reader) the ring goes back to
	// the allocator and the next segment's pass 1 is queued on the second stream, to run beside this segment's resolve and CRC and
	// the parse of its window
	const uint64_t pos = kind == GZS_LAST ? len_ * 8 : gzs_next_bit(p.base * 8, &next, 0);
	const uint64_t in_next = in_used_ + (pos - pos_) / 8, out_next = out_made_ + total;
	const uint64_t seg_next = gzs_seg_len(cap, in_next, out_next);
	size_t peak = s.peak;
	if (kind == GZS_STOP) {
		GZ_CUDA(cudaStreamSynchronize(st_));            // (nothing on the main stream uses memory the prefetch may be given)
		s.put(p.ring), p.ring = nullptr;
		const uint64_t b = pos >> 3;
		pre_ = p1_launch(pos, seg_next < len_ - b ? seg_next : len_ - b, false, st2_); // (a read error: the next fill reads again)
		if (pre_ && s.now + pre_->s.peak > peak) peak = s.now + pre_->s.peak;
	}
	uint64_t *m_end = s.get<uint64_t>(members + 1);
	uint32_t *m_crc = s.get<uint32_t>(members + 1), *m_isize = s.get<uint32_t>(members + 1);
	k_gz_resolve<<<(nc + 31) / 32, 32, 0, st_>>>(p.gz, n, p.starts, nu, chain, nc, off, mbase, p.ust, p.land, p.olen, p.nmem, win, valid,
	                                             dst, m_end, m_crc, m_isize, d_sc, p.hdr);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev_[4], st_));
	const uint64_t n_seg = (total + GZ_SEG - 1) / GZ_SEG;
	uint32_t *seg_crc = s.get<uint32_t>(n_seg);
	if (n_seg) { k_gz_crc_seg<<<(unsigned)((n_seg + 255) / 256), 256, 0, st_>>>(dst, total, GZ_SEG, seg_crc); GZ_CUDA(cudaGetLastError()); }
	k_gz_crc_member<<<(unsigned)members + 1, 128, 0, st_>>>(dst, GZ_SEG, seg_crc, m_end, m_crc, m_isize, d_sc, (uint32_t)members, total, carry_, carry_ + 2);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev_[5], st_));
	fetch();
	GZ_CUDA(cudaEventElapsedTime(&ms[3], ev_[2], ev_[3]));
	GZ_CUDA(cudaEventElapsedTime(&ms[4], ev_[3], ev_[4]));
	GZ_CUDA(cudaEventElapsedTime(&ms[5], ev_[4], ev_[5]));
	sum.ms_window += ms[3], sum.ms_resolve += ms[4], sum.ms_crc += ms[5];
	sum.n_chain += nc, sum.n_confirmed += h_sc[GS_CONF], sum.n_members += members;
	if (s.peak > peak) peak = s.peak;
	if (peak > sum.scratch_peak) sum.scratch_peak = peak;
	if (h_sc[GS_ERR]) return GZ_REJECT;
	// hand on: the window after the last unit taken, the CRC of the member left open, the next unit's bit
	GZ_CUDA(cudaMemcpyAsync(hist_, win + (size_t)nc * INF_WIN, INF_WIN, cudaMemcpyDeviceToDevice, st_));
	GZ_CUDA(cudaMemcpyAsync(valid_, valid + nc, sizeof(uint32_t), cudaMemcpyDeviceToDevice, st_));
	GZ_CUDA(cudaMemcpyAsync(carry_, carry_ + 2, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st_));
	hdr_ = false;
	need_ = gzs_need_after(need_next, cap, total);
	in_used_ = in_next, out_made_ = out_next, next_seg_ = seg_next, sum.out_len += total;
	pos_ = pos;
	if (kind == GZS_LAST) done_ = true;
	return (int64_t)total;
}
