/* main.c -- the miniasm-b200 command line: same options, step order, stderr chatter and output formats as
 * the reference driver (main.c:32-211), with every step of the hot path running on the GPU through the fused
 * C ABI (include/miniasm_b200.h).  Usage: miniasm-b200 [options] <in.paf>
 * Extra environment: MINIASM_B200_DEVICE=<cuda ordinal> (first device), MINIASM_B200_GPUS=<N>: the default pipeline
 * (no -R/-1/-2/-S/-f, -p ug|sg) hash-sharded over N GPUs of this node -- one thread and one context per GPU, the PAF cut
 * into N byte ranges at line ends, NCCL inside the library (SURVEY.md 8e).  Same bytes on stdout as with one GPU. */
#include <unistd.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>
#include <pthread.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <zlib.h>
#include "miniasm_b200.h"

#define MAB_VERSION "0.3-r179"   /* tracks the reference release whose output it reproduces */

static void usage(const ma_opt_t *o, const char *outfmt)
{
	fprintf(stderr, "Usage: miniasm-b200 [options] <in.paf>\n");
	fprintf(stderr, "Options:\n");
	fprintf(stderr, "  Pre-selection:\n");
	fprintf(stderr, "    -R          prefilter clearly contained reads (2-pass required)\n");
	fprintf(stderr, "    -m INT      min match length [%d]\n", o->min_match);
	fprintf(stderr, "    -i FLOAT    min identity [%.2g]\n", o->min_iden);
	fprintf(stderr, "    -s INT      min span [%d]\n", o->min_span);
	fprintf(stderr, "    -c INT      min coverage [%d]\n", o->min_dp);
	fprintf(stderr, "  Overlap:\n");
	fprintf(stderr, "    -o INT      min overlap [same as -s]\n");
	fprintf(stderr, "    -h INT      max over hang length [%d]\n", o->max_hang);
	fprintf(stderr, "    -I FLOAT    min end-to-end match ratio [%.2g]\n", o->int_frac);
	fprintf(stderr, "  Layout:\n");
	fprintf(stderr, "    -g INT      max gap differences between reads for trans-reduction [%d]\n", o->gap_fuzz);
	fprintf(stderr, "    -d INT      max distance for bubble popping [%d]\n", o->bub_dist);
	fprintf(stderr, "    -e INT      small unitig threshold [%d]\n", o->max_ext);
	fprintf(stderr, "    -f FILE     read sequences []\n");
	fprintf(stderr, "    -n INT      rounds of short overlap removal [%d]\n", o->n_rounds + 1);
	fprintf(stderr, "    -r FLOAT[,FLOAT]\n");
	fprintf(stderr, "                max and min overlap drop ratio [%.2g,%.2g]\n", o->max_ovlp_drop_ratio, o->min_ovlp_drop_ratio);
	fprintf(stderr, "    -F FLOAT    aggressive overlap drop ratio in the end [%.2g]\n", o->final_ovlp_drop_ratio);
	fprintf(stderr, "  Miscellaneous:\n");
	fprintf(stderr, "    -p STR      output information: bed, paf, sg or ug [%s]\n", outfmt);
	fprintf(stderr, "    -b          both directions of an arc are present in input\n");
	fprintf(stderr, "    -1          skip 1-pass read selection\n");
	fprintf(stderr, "    -2          skip 2-pass read selection\n");
	fprintf(stderr, "    -V          print version number\n");
	fprintf(stderr, "\nSee miniasm.1 of the reference for a detailed description of the command-line options.\n");
}

/* ---- MINIASM_B200_GPUS=N: one thread per GPU ------------------------------------------------------------------ */
typedef struct {
	int rank, world, device, bi_dir;
	const ma_opt_t *opt;
	const char *text;            /* this rank's byte range of the PAF */
	size_t len;
	const void *nccl_id;
	mab_ctx_t *ctx;
} rank_job_t;

static void *rank_main(void *p)
{
	rank_job_t *j = (rank_job_t*)p;
	j->ctx = mab_create(j->device);
	mab_shard_init(j->ctx, j->rank, j->world, j->nccl_id);
	mab_load_ingest_text_sharded(j->ctx, j->text, j->len, j->opt->min_span, j->opt->min_match, j->bi_dir); /* chunks parsed while the next ones are copied */
	mab_select_sharded(j->ctx, j->opt);
	mab_layout_sharded(j->ctx, j->opt);
	return 0;
}

/* the whole PAF in host memory: plain files are mapped, gzip / stdin are inflated into a heap buffer */
static char *slurp(const char *fn, size_t *len, int *mapped)
{
	unsigned char magic[2] = {0, 0};
	int fd = strcmp(fn, "-") ? open(fn, O_RDONLY) : -1;
	struct stat sb;
	*mapped = 0;
	if (fd >= 0 && fstat(fd, &sb) == 0 && S_ISREG(sb.st_mode) && sb.st_size > 0 && pread(fd, magic, 2, 0) == 2 && !(magic[0] == 0x1f && magic[1] == 0x8b)) {
		char *m = (char*)mmap(0, (size_t)sb.st_size, PROT_READ, MAP_PRIVATE | MAP_POPULATE, fd, 0);
		close(fd);
		if (m != MAP_FAILED) { *len = (size_t)sb.st_size, *mapped = 1; return m; }
		fd = -1;
	}
	if (fd >= 0) close(fd);
	{
		gzFile fp = strcmp(fn, "-") ? gzopen(fn, "r") : gzdopen(fileno(stdin), "r");
		size_t n = 0, m = 1 << 24;
		char *buf;
		int r;
		if (fp == 0) return 0;
		gzbuffer(fp, 1 << 20);
		buf = (char*)malloc(m);
		while ((r = gzread(fp, buf + n, (unsigned)(m - n < (1u << 30) ? m - n : (1u << 30)))) > 0) {
			n += (size_t)r;
			if (n == m) buf = (char*)realloc(buf, m <<= 1);
		}
		gzclose(fp);
		*len = n;
		return buf;
	}
}

/* steps 1-4 on `world` GPUs; returns rank 0's context (holding the same reduced graph a single GPU would) */
static mab_ctx_t *run_sharded(const char *fn, const ma_opt_t *opt, int bi_dir, int world, int device0)
{
	char id[128];
	size_t len = 0, cut[65];
	int r, mapped = 0;
	char *text = slurp(fn, &len, &mapped);
	pthread_t tid[64];
	rank_job_t job[64];
	mab_ctx_t *ctx0;
	if (text == 0) {
		fprintf(stderr, "[E::%s] could not open PAF file %s\n", "ma_hit_read", fn);
		exit(1);
	}
	cut[0] = 0;
	for (r = 1; r < world; ++r) { /* byte ranges in rank order, each ending after a newline */
		size_t p = len / world * r;
		const char *q;
		if (p < cut[r - 1]) p = cut[r - 1];
		q = p < len ? (const char*)memchr(text + p, '\n', len - p) : 0;
		cut[r] = q ? (size_t)(q - text) + 1 : len;
	}
	cut[world] = len;
	mab_nccl_unique_id(id);
	for (r = 0; r < world; ++r) {
		job[r].rank = r, job[r].world = world, job[r].device = device0 + r, job[r].bi_dir = bi_dir, job[r].opt = opt;
		job[r].text = text + cut[r], job[r].len = cut[r + 1] - cut[r], job[r].nccl_id = id, job[r].ctx = 0;
		pthread_create(&tid[r], 0, rank_main, &job[r]);
	}
	for (r = 0; r < world; ++r) pthread_join(tid[r], 0);
	if (mapped) munmap(text, len); else free(text);
	ctx0 = job[0].ctx;
	for (r = 1; r < world; ++r) mab_destroy(job[r].ctx);
	return ctx0;
}

/* MINIASM_B200_INGEST=auto: does Step 1 take the windowed ingest?  Only for a plain regular file whose text and line arrays
 * (what the resident ingest holds beside the hits: the padded text, a line start and a 32-byte record per estimated line) would
 * take more than half of the free device memory -- inputs the resident ingest cannot hold.  The half is a guess, not a measurement. */
static int auto_windowed(mab_ctx_t *ctx, const char *fn)
{
	struct stat sb;
	unsigned char magic[2] = {0, 0};
	int fd, plain;
	size_t len;
	if (strcmp(fn, "-") == 0 || (fd = open(fn, O_RDONLY)) < 0) return 0;
	plain = fstat(fd, &sb) == 0 && S_ISREG(sb.st_mode) && !(pread(fd, magic, 2, 0) == 2 && magic[0] == 0x1f && magic[1] == 0x8b);
	close(fd);
	if (!plain) return 0;
	len = (size_t)sb.st_size;
	return len / 8 * 9 + 40 * (len / 24 + 1024) > mab_mem_free(ctx) / 2;
}

int main(int argc, char *argv[])
{
	ma_opt_t opt;
	int i, c, stage = 100, no_first = 0, no_second = 0, bi_dir = 1, o_set = 0, no_cont = 0, device = 0, n_gpus = 1, sharded_done = 0, gpu_seq = 0;
	int windowed = -1;           /* MINIASM_B200_INGEST: 1 windowed, 0 resident, -1 auto */
	size_t window_bytes = 0;     /* MINIASM_B200_WINDOW (0: the library's default) */
	const char *fn_reads = 0, *outfmt = "ug", *env;
	mab_ctx_t *ctx;
	FILE *out = stdout;          /* where the GFA goes */
	sdict_t *d = 0;
	ma_sub_t *sub = 0;

	ma_opt_init(&opt);
	while ((c = getopt(argc, argv, "n:m:s:c:S:i:d:g:o:h:I:r:f:e:p:12VBRbF:")) >= 0) {
		switch (c) {
			case 'm': opt.min_match = atoi(optarg); break;
			case 'i': opt.min_iden = atof(optarg); break;
			case 's': opt.min_span = atoi(optarg); break;
			case 'c': opt.min_dp = atoi(optarg); break;
			case 'o': opt.min_ovlp = atoi(optarg), o_set = 1; break;
			case 'S': stage = atoi(optarg); break;
			case 'd': opt.bub_dist = atoi(optarg); break;
			case 'g': opt.gap_fuzz = atoi(optarg); break;
			case 'h': opt.max_hang = atoi(optarg); break;
			case 'I': opt.int_frac = atof(optarg); break;
			case 'e': opt.max_ext = atoi(optarg); break;
			case 'f': fn_reads = optarg; break;
			case 'p': outfmt = optarg; break;
			case '1': no_first = 1; break;
			case '2': no_second = 1; break;
			case 'n': opt.n_rounds = atoi(optarg) - 1; break;
			case 'B': bi_dir = 1; break;
			case 'b': bi_dir = 0; break;
			case 'R': no_cont = 1; break;
			case 'F': opt.final_ovlp_drop_ratio = atof(optarg); break;
			case 'V': printf("%s\n", MAB_VERSION); return 0;
			case 'r': {
				char *s;
				opt.max_ovlp_drop_ratio = strtod(optarg, &s);
				if (*s == ',') opt.min_ovlp_drop_ratio = strtod(s + 1, &s);
				break; }
		}
	}
	if (o_set == 0) opt.min_ovlp = opt.min_span;
	if (argc == optind) { usage(&opt, outfmt); return 1; }

	sys_init();
	if ((env = getenv("MINIASM_B200_DEVICE")) != 0) device = atoi(env);
	if ((env = getenv("MINIASM_B200_GPUS")) != 0) n_gpus = atoi(env);
	if (n_gpus > 64) n_gpus = 64;
	if (n_gpus > 1 && (no_cont || no_first || no_second || stage < 100 || fn_reads || (strcmp(outfmt, "ug") && strcmp(outfmt, "sg")))) {
		fprintf(stderr, "[W::%s] MINIASM_B200_GPUS=%d covers the default pipeline (-p ug|sg without -R/-1/-2/-S/-f): running on one GPU\n", __func__, n_gpus);
		n_gpus = 1;
	}
	if ((env = getenv("MINIASM_B200_INGEST")) != 0) windowed = strcmp(env, "windowed") == 0 ? 1 : strcmp(env, "resident") == 0 ? 0 : -1;
	if ((env = getenv("MINIASM_B200_WINDOW")) != 0) window_bytes = (size_t)strtoull(env, 0, 10);
	if (windowed == 1 && (no_cont || n_gpus > 1 || strcmp(argv[optind], "-") == 0)) { /* (auto never picks it for these) */
		fprintf(stderr, "[W::%s] MINIASM_B200_INGEST=windowed does not cover %s: the PAF text is loaded whole\n", __func__,
		        no_cont ? "-R" : n_gpus > 1 ? "MINIASM_B200_GPUS" : "standard input, which cannot be read twice");
		windowed = 0;
	}
	if (no_cont || n_gpus > 1) windowed = 0;
	if (n_gpus > 1) { /* steps 1-4 sharded; what follows (unitigs, output) runs on rank 0's context as in a single-GPU run */
		/* stdout carries the GFA and NCCL prints its version banner (NCCL_DEBUG=VERSION) there: the GFA keeps the original
		 * descriptor, everything else that writes to fd 1 from here on lands on stderr */
		int fd;
		fflush(stdout);
		fd = dup(1);
		if (fd >= 0 && dup2(2, 1) >= 0) out = fdopen(fd, "w");
		if (out == 0) out = stdout;
		fprintf(stderr, "[M::%s] ===> Step 1: reading read mappings <===\n", __func__);
		fprintf(stderr, "[M::%s] ===> Step 2: 1-pass (crude) read selection <===\n", __func__);
		fprintf(stderr, "[M::%s] ===> Step 3: 2-pass (fine) read selection <===\n", __func__);
		fprintf(stderr, "[M::%s] ===> Step 4: graph cleaning <===\n", __func__);
		ctx = run_sharded(argv[optind], &opt, bi_dir, n_gpus, device);
		sharded_done = 1;
	} else ctx = mab_create(device);
	/* -f: the reads file starts streaming into HBM now, on its own thread and stream, behind the graph stages */
	if (fn_reads && strcmp(outfmt, "ug") == 0 && !((env = getenv("MAB_GPU_SEQ")) != 0 && atoi(env) == 0)) mab_reads_prefetch(ctx, fn_reads), gpu_seq = 1;

	if (sharded_done) {
	} else if (no_cont) { /* -R: Step 0 (contained-read prefilter) and Step 1 share one pass over the text in HBM */
		fprintf(stderr, "[M::%s] ===> Step 0: removing contained reads <===\n", __func__);
		if (mab_load_paf_file(ctx, argv[optind]) < 0) {
			fprintf(stderr, "[E::%s] could not open PAF file %s\n", "ma_hit_no_cont", argv[optind]);
			exit(1);
		}
		mab_ingest_nocont(ctx, opt.min_span, opt.min_match, bi_dir, opt.max_hang, opt.int_frac);
	} else {
		int rc = -2;                 /* -2: the windowed ingest did not run */
		fprintf(stderr, "[M::%s] ===> Step 1: reading read mappings <===\n", __func__);
		if (windowed < 0) windowed = auto_windowed(ctx, argv[optind]);
		if (windowed) rc = mab_ingest_file_windowed(ctx, argv[optind], window_bytes, opt.min_span, opt.min_match, bi_dir);
		if (rc == -2 && windowed) fprintf(stderr, "[W::%s] %s cannot be read twice: the PAF text is loaded whole\n", __func__, argv[optind]);
		if (rc == -1 || (rc == -2 && mab_load_paf_file(ctx, argv[optind]) < 0)) {
			fprintf(stderr, "[E::%s] could not open PAF file %s\n", "ma_hit_read", argv[optind]);
			exit(1);
		}
		if (rc == -2) mab_ingest(ctx, opt.min_span, opt.min_match, bi_dir);
	}

	if (!sharded_done) mab_select(ctx, &opt, no_first, no_second, stage); /* prints the Step 2 / Step 3 banners where the reference does */

	if (strcmp(outfmt, "bed") == 0) {
		mab_write_bed(ctx, out);     /* print_subs, formatted on the GPU; nothing when no read selection ran (-1 -2) */
	} else if (strcmp(outfmt, "paf") == 0) {
		mab_write_paf(ctx, out);     /* print_hits, likewise */
	} else if (strcmp(outfmt, "ug") == 0 || strcmp(outfmt, "sg") == 0) {
		/* no -f: the GFA text is formatted on the GPU and copied down once (MAB_GPU_GFA=0: host structs + ma_ug_print) */
		const int gpu_gfa = strcmp(outfmt, "ug") == 0 && !fn_reads && !((env = getenv("MAB_GPU_GFA")) != 0 && atoi(env) == 0);
		if (!sharded_done) {
			fprintf(stderr, "[M::%s] ===> Step 4: graph cleaning <===\n", __func__);
			mab_layout(ctx, &opt, stage);
		}
		if (strcmp(outfmt, "ug") == 0) {
			ma_ug_t *ug;
			fprintf(stderr, "[M::%s] ===> Step 5: generating unitigs <===\n", __func__);
			mab_unitigs(ctx);
			if (gpu_gfa) {
				mab_write_gfa(ctx, out);
			} else if (gpu_seq && mab_write_gfa_reads(ctx, out, fn_reads) != -2) {
				/* ma_ug_seq + ma_ug_print on the GPU (MAB_GPU_SEQ=0, or a reads file that is neither FASTA-like nor 4-line FASTQ: host path below) */
			} else {
				d = mab_export_dict(ctx), sub = mab_export_sub(ctx);
				ug = mab_export_ug(ctx);
				if (fn_reads) ma_ug_seq(ug, d, sub, fn_reads);
				ma_ug_print(ug, d, sub, out);
				ma_ug_destroy(ug);
			}
		} else {
			mab_write_sg(ctx, out);      /* ma_sg_print, formatted on the GPU */
		}
	}
	if (out != stdout) fclose(out);
	free(sub);
	if (d) sd_destroy(d);
	mab_destroy(ctx);

	fprintf(stderr, "[M::%s] Version: %s\n", __func__, MAB_VERSION);
	fprintf(stderr, "[M::%s] CMD:", __func__);
	for (i = 0; i < argc; ++i) fprintf(stderr, " %s", argv[i]);
	fprintf(stderr, "\n[M::%s] Real time: %.3f sec; CPU: %.3f sec\n", __func__, sys_realtime(), sys_cputime());
	return 0;
}
