/*
 * tools/find_hard_phases.c — search float pairs (re, im) whose atan2(im, re) lies within a few double ulps of a float
 * rounding boundary (the midpoint between two neighbouring floats).  Those are the only samples on which an atan2
 * evaluated in double with an error of an ulp or two can narrow to the wrong float, and the ones on which
 * vdl2_phase_fast (dumpvdl2_b200/csrc/vdl2_fastmath.cuh) must hand over to its fall-back.
 *
 *   cc -O2 -std=c11 -pthread tools/find_hard_phases.c -o find_hard_phases -lm
 *   find_hard_phases SEED CLASS BLOCKS [THREADS]      (one block = 2^20 draws)
 *
 * Each candidate is printed as "class block index re_bits im_bits dist": dist is the signed distance of the 64-bit
 * long double atan2l from the midpoint, in units of the last bit of a double at the midpoint (positive: above).
 * Every block draws from its own generator seeded with (SEED, CLASS, block), so the set of candidates depends on
 * the seed and the number of blocks only, not on the number of threads or on their timing; sort the output.
 * tests/golden/make_phase_hard.py runs this tool and confirms every candidate at 200 bits.
 *
 * Classes (the draws; every class keeps the candidates within HARD_ULPS of a midpoint, except the guard class):
 *   0 random      |re|, |im| over 2^-12..1, uniform binade (decimated-sample levels), random signs: all eight octants
 *   1 near_pi     re < 0, |im| < 1e-6 |re|: results next to +-pi, which leave the fast path by its range test
 *   2 near_pio2   |re| < 1e-6 |im|: results next to +-pi/2 (same)
 *   3 break       min/max within 2^-20 of a break point (k + 1/2)/8, where the fast path picks one of two k
 *   4 pow2        results within 2^-10 (relative) of a power of two 2^1 .. 2^-12, where the float spacing halves
 *   5 guard       draws as in class 0 whose atan2 lies 400..700 units of the last double bit from the
 *                 midpoint: just inside and just outside the fast path's 512-unit guard (its error is ~16 units)
 */
#include <math.h>
#include <pthread.h>
#include <stdbool.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define BLOCK_DRAWS (1u << 20)
#define HARD_ULPS 4.0L        /* classes 0-4: |dist| < 4 */
#define GUARD_LO 400.0L       /* class 5: 400 <= |dist| < 700 */
#define GUARD_HI 700.0L
#define PREFILTER_SLACK 8.0   /* glibc's double atan2 is within an ulp of the exact value */
#define PIO2 0x1.921fb54442d18p+0
#define PI 0x1.921fb54442d18p+1

static uint64_t g_seed;
static int g_class;
static uint64_t g_blocks;
static uint64_t g_next;
static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;

static uint64_t splitmix(uint64_t *s) {
	uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	return z ^ (z >> 31);
}
static double unif(uint64_t *s) { return (double)(splitmix(s) >> 11) * 0x1p-53; }
/* 2^-12 .. 1: a uniform binade, then a uniform float in it */
static float level(uint64_t *s) { const uint64_t z = splitmix(s); return ldexpf(1.0f + (float)(z & 0x7FFFFF) * 0x1p-23f, -1 - (int)((z >> 23) % 12)); }
static float sgn(uint64_t *s, float x) { return (splitmix(s) & 1) ? -x : x; }
static uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* signed distance of x from the nearest float midpoint, in units of the last bit of a double at that midpoint */
static long double midpoint_dist(long double x) {
	const float f = (float)x;
	const float g = nextafterf(f, x > (long double)f ? INFINITY : -INFINITY);
	const long double mid = ((long double)f + (long double)g) / 2;
	const long double ulp = ldexpl(1.0L, ilogbl(mid) - 52);
	return (x - mid) / ulp;
}

static bool draw(uint64_t *s, float *re, float *im) {
	switch(g_class) {
	case 0: case 5:
		*re = sgn(s, level(s)); *im = sgn(s, level(s));
		return true;
	case 1: {
		const float r = level(s);
		const float q = (float)(1e-6 * exp2(-20.0 * unif(s)));
		*re = -r; *im = sgn(s, r * q);
		return *im != 0.0f && fabsf(*im) < 1e-6f * r;
	}
	case 2: {
		const float r = level(s);
		const float q = (float)(1e-6 * exp2(-20.0 * unif(s)));
		*im = sgn(s, r); *re = sgn(s, r * q);
		return *re != 0.0f && fabsf(*re) < 1e-6f * r;
	}
	case 3: {
		const float mx = level(s);
		const int k = (int)(splitmix(s) % 8);
		const float mn = (float)((double)mx * (k + 0.5) / 8.0 * (1.0 + (2.0 * unif(s) - 1.0) * 0x1p-20));
		const double q = (double)mn / (double)mx;
		if(fabs(q - (k + 0.5) / 8.0) > 0x1p-20) return false;
		if(splitmix(s) & 1) { *re = sgn(s, mx); *im = sgn(s, mn); } else { *re = sgn(s, mn); *im = sgn(s, mx); }
		return true;
	}
	case 4: {
		const int j = 1 - (int)(splitmix(s) % 14);                  /* 2^1 .. 2^-12 */
		const double th = ldexp(1.0 + (2.0 * unif(s) - 1.0) * 0x1p-10, j);
		const double r = exp2(-12.0 * unif(s));
		*re = (float)(r * cos(th)); *im = sgn(s, (float)(r * sin(th)));
		return *re != 0.0f && *im != 0.0f;
	}
	}
	return false;
}

static void *worker(void *arg) {
	(void)arg;
	const long double lo = g_class == 5 ? GUARD_LO : 0.0L, hi = g_class == 5 ? GUARD_HI : HARD_ULPS;
	for(;;) {
		pthread_mutex_lock(&g_lock);
		const uint64_t b = g_next++;
		pthread_mutex_unlock(&g_lock);
		if(b >= g_blocks) return NULL;
		uint64_t s = g_seed ^ ((uint64_t)g_class << 56) ^ (b * 0xD1B54A32D192ED03ull);
		char out[8192];
		size_t used = 0;
		out[0] = 0;
		for(uint32_t i = 0; i < BLOCK_DRAWS && used < sizeof out - 128; i++) {
			float re, im;
			if(!draw(&s, &re, &im)) continue;
			/* a draw of class 0 or 5 serves four octants: with mx = max(|re|, |im|), mn = min and a = atan2(mn, mx), the
			 * results a, pi/2 - a, pi/2 + a and pi - a belong to (mx, mn), (mn, mx), (-mn, mx) and (-mx, mn); the sign of
			 * im then picks the half plane.  The other classes keep their own draw. */
			const int n_fold = g_class == 0 || g_class == 5 ? 4 : 1;
			const float mx = fmaxf(fabsf(re), fabsf(im)), mn = fminf(fabsf(re), fabsf(im));
			const float sg = im < 0.0f ? -1.0f : 1.0f;
			const double a0 = atan2((double)mn, (double)mx);
			for(int o = 0; o < n_fold; o++) {
				float r = re, m = im;
				double a;
				switch(n_fold == 1 ? -1 : o) {
				case 0: r = mx; m = sg * mn; a = a0; break;
				case 1: r = mn; m = sg * mx; a = PIO2 - a0; break;
				case 2: r = -mn; m = sg * mx; a = PIO2 + a0; break;
				case 3: r = -mx; m = sg * mn; a = PI - a0; break;
				default: a = atan2((double)im, (double)re); break;
				}
				/* prefilter in double (glibc's atan2 is within an ulp, a fold adds one), confirm with the 64-bit atan2l */
				const float f = (float)a;
				const float g = nextafterf(f, a > (double)f ? INFINITY : -INFINITY);
				const double mid = ((double)f + (double)g) / 2;
				const double da = fabs(a - mid) / ldexp(1.0, ilogb(mid) - 52);
				if(da > (double)hi + PREFILTER_SLACK || da < (double)lo - PREFILTER_SLACK) continue;
				const long double d = midpoint_dist(atan2l((long double)m, (long double)r));
				if(fabsl(d) >= hi || fabsl(d) < lo) continue;
				used += (size_t)snprintf(out + used, sizeof out - used, "%d %llu %u %08x %08x %.6Lf\n", g_class,
						(unsigned long long)b, i, fbits(r), fbits(m), d);
			}
		}
		pthread_mutex_lock(&g_lock);
		fputs(out, stdout);
		fflush(stdout);
		pthread_mutex_unlock(&g_lock);
	}
}

int main(int argc, char **argv) {
	if(argc < 4) { fprintf(stderr, "usage: %s SEED CLASS BLOCKS [THREADS]\n", argv[0]); return 2; }
	g_seed = strtoull(argv[1], NULL, 0);
	g_class = atoi(argv[2]);
	g_blocks = strtoull(argv[3], NULL, 0);
	const int nt = argc > 4 ? atoi(argv[4]) : 8;
	if(g_class < 0 || g_class > 5 || nt < 1 || nt > 256) return 2;
	pthread_t th[256];
	for(int t = 0; t < nt; t++) pthread_create(&th[t], NULL, worker, NULL);
	for(int t = 0; t < nt; t++) pthread_join(th[t], NULL);
	return 0;
}
