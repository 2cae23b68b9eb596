/* bitnetmcu_b200_concurrency.c -- Inference() called from many threads at once (plain C, gcc -pthread).
 *
 *     concurrency <dll> <digits.bin> <threads> <calls per thread>
 *
 * dlopen()s <dll> -- the gcc-built shim of this library (host/bitnetmcu_b200_dll.c) or the reference's own Bitnet_inf.dll --
 * and runs <threads> pthreads that each call `uint32_t Inference(int8_t *input)` (/root/reference/BitNetMCU_MNIST_dll.c:24-26)
 * <calls per thread> times, one 16x16 image per call, over the 256-byte images of <digits.bin>.  The threads warm up, meet at a
 * barrier, then run; each call is timed on its own.  Prints one JSON line: calls per second over the whole run, the median and
 * 99th percentile of the microseconds per call, the labels of the first ten images (one thread, before the run) and the number
 * of calls in the run whose label differs from that one-thread label of the same image. */
#include <dlfcn.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

typedef uint32_t (*inference_fn)(int8_t *);

enum { kMaxImages = 64, kWarmup = 20 };
static int8_t g_imgs[kMaxImages][256];
static uint32_t g_want[kMaxImages];
static size_t g_n_img;
static inference_fn g_fn;
static long g_calls;
static pthread_barrier_t g_start;

typedef struct {
    int index;
    double *us;        /* [g_calls] microseconds per call */
    long mismatches;
} worker;

static double now_us(void) {
    struct timespec t;
    clock_gettime(CLOCK_MONOTONIC, &t);
    return t.tv_sec * 1e6 + t.tv_nsec / 1e3;
}

static void *run(void *arg) {
    worker *w = (worker *)arg;
    int8_t img[256];   /* the thread's own copy: each call reads its image from the caller's memory */
    for (int i = 0; i < kWarmup; i++) {
        memcpy(img, g_imgs[(w->index + i) % g_n_img], 256);
        g_fn(img);
    }
    pthread_barrier_wait(&g_start);
    for (long i = 0; i < g_calls; i++) {
        const size_t k = (size_t)(w->index * 7 + i) % g_n_img;
        memcpy(img, g_imgs[k], 256);
        const double t0 = now_us();
        const uint32_t label = g_fn(img);
        w->us[i] = now_us() - t0;
        w->mismatches += label != g_want[k];
    }
    return NULL;
}

static int by_value(const void *a, const void *b) {
    const double x = *(const double *)a, y = *(const double *)b;
    return (x > y) - (x < y);
}

int main(int argc, char **argv) {
    if (argc < 5) { fprintf(stderr, "usage: %s <dll> <digits.bin> <threads> <calls per thread>\n", argv[0]); return 2; }
    void *h = dlopen(argv[1], RTLD_NOW);
    if (!h) { fprintf(stderr, "dlopen: %s\n", dlerror()); return 1; }
    g_fn = (inference_fn)dlsym(h, "Inference");
    if (!g_fn) { fprintf(stderr, "no Inference() in %s\n", argv[1]); return 1; }
    FILE *f = fopen(argv[2], "rb");
    if (!f) { perror(argv[2]); return 1; }
    g_n_img = fread(g_imgs, 256, kMaxImages, f);
    fclose(f);
    if (g_n_img == 0) return 1;
    const int threads = atoi(argv[3]);
    g_calls = atol(argv[4]);
    if (threads < 1 || g_calls < 1) { fprintf(stderr, "threads and calls must be >= 1\n"); return 2; }
    for (size_t i = 0; i < g_n_img; i++) g_want[i] = g_fn(g_imgs[i]);   /* one thread: the labels every call must return */

    worker *w = calloc((size_t)threads, sizeof(worker));
    double *us = malloc((size_t)threads * (size_t)g_calls * sizeof(double));
    pthread_t *tid = malloc((size_t)threads * sizeof(pthread_t));
    if (!w || !us || !tid) { fprintf(stderr, "out of memory\n"); return 1; }
    pthread_barrier_init(&g_start, NULL, (unsigned)threads + 1);
    for (int t = 0; t < threads; t++) {
        w[t].index = t;
        w[t].us = us + (size_t)t * (size_t)g_calls;
        if (pthread_create(&tid[t], NULL, run, &w[t]) != 0) { fprintf(stderr, "pthread_create failed\n"); return 1; }
    }
    pthread_barrier_wait(&g_start);
    const double t0 = now_us();
    long mismatches = 0;
    for (int t = 0; t < threads; t++) {
        pthread_join(tid[t], NULL);
        mismatches += w[t].mismatches;
    }
    const double wall = now_us() - t0;
    const size_t total = (size_t)threads * (size_t)g_calls;
    qsort(us, total, sizeof(double), by_value);
    printf("{\"threads\": %d, \"calls\": %zu, \"calls_per_s\": %.1f, \"p50_us\": %.2f, \"p99_us\": %.2f, \"labels\": \"", threads, total,
           total / (wall / 1e6), us[total / 2], us[(size_t)(total * 0.99)]);
    for (size_t i = 0; i < 10 && i < g_n_img; i++) printf("%s%u", i ? "," : "", g_want[i]);
    printf("\", \"mismatches\": %ld}\n", mismatches);
    pthread_barrier_destroy(&g_start);
    free(tid);
    free(us);
    free(w);
    return 0;
}
