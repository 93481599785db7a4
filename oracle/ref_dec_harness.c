/*
 * oracle/ref_dec_harness.c — TEST INFRASTRUCTURE ONLY (never linked into libvdl2gpu.so).
 *
 * Driver for the UNMODIFIED reference demodulator on decimated samples.  demod() is static in the reference's
 * src/demod.c, so that file is compiled inside this translation unit (#include, from where it lies; see
 * oracle/Makefile) and demod() is called directly, one channel after the other, sample by sample: the loop body of
 * process_samples after its decimation step (reference src/demod.c:322-328).  The frame capture, the globals and the
 * stand-ins are ref_harness.c's.
 *
 * Usage: vdl2_ref_dec --freqs f0,f1,... [--max-ppm X] FILE
 *        FILE: float32 decimated samples, time-major [n][channels][2] (re, im)
 * Output (stdout): ref_harness.c's FRAME lines, then  DEC channels=C samples=N frames=F
 */
#define REF_HARNESS_NO_MAIN
#include "ref_harness.c"
#include "demod.c"

int main(int argc, char **argv) {
	char const *freqs_s = NULL, *file = NULL;
	memset(&Config, 0, sizeof(Config));
	for(int i = 1; i < argc; i++) {
		if(!strcmp(argv[i], "--freqs") && i+1 < argc) freqs_s = argv[++i];
		else if(!strcmp(argv[i], "--max-ppm") && i+1 < argc) Config.max_ppm = strtof(argv[++i], NULL);
		else if(argv[i][0] != '-') file = argv[i];
		else { fprintf(stderr, "unknown option %s\n", argv[i]); return 2; }
	}
	if(!file || !freqs_s) { fprintf(stderr, "need --freqs and FILE\n"); return 2; }
	uint32_t *freqs = NULL;
	{
		char *dup = strdup(freqs_s), *save = NULL;
		for(char *t = strtok_r(dup, ",", &save); t; t = strtok_r(NULL, ",", &save)) {
			freqs = realloc(freqs, (num_channels + 1) * sizeof(uint32_t));
			freqs[num_channels++] = strtoul(t, NULL, 10);
		}
		free(dup);
	}
	chan_freqs = freqs;
	FILE *f = fopen(file, "rb");
	if(!f) { perror(file); return 2; }
	fseek(f, 0, SEEK_END);
	long fsize = ftell(f);
	fseek(f, 0, SEEK_SET);
	size_t n_float = (size_t)fsize / sizeof(float);
	float *dec = malloc(n_float ? n_float * sizeof(float) : 1);
	if(fread(dec, sizeof(float), n_float, f) != n_float) { perror("fread"); return 2; }
	fclose(f);
	size_t n_dec = n_float / (2 * (size_t)num_channels);

	/* what the reference initialises for the demodulator and the decoder: src/dumpvdl2.c:1086-1153.  The channels are
	 * not offset-tuned (centre == channel frequency): the front end is not run here. */
	captures = calloc(num_channels, sizeof(*captures));
	if(rs_init() < 0) { fprintf(stderr, "rs_init failed\n"); return 3; }
	avlc_decoder_init();
	demod_sync_init();
	for(int i = 0; i < num_channels; i++) {
		vdl2_channel_t *v = vdl2_channel_init(freqs[i], freqs[i], SYMBOL_RATE * SPS, 1);
		tl_chan = i;
		for(size_t n = 0; n < n_dec; n++) {
			const float *d = &dec[(n * (size_t)num_channels + (size_t)i) * 2];
			demod(v, d[0], d[1]);
		}
	}
	size_t nframes = print_captures();
	printf("DEC channels=%d samples=%zu frames=%zu\n", num_channels, n_dec, nframes);
	fflush(stdout);
	return 0;
}
