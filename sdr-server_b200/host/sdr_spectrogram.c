/*
 * host/sdr_spectrogram.c -- the reference's offline spectrogram tool (src/spectrogram/) on the batch group: it reads
 * an IQ recording in cu8, cs16 or cf32 (optionally gzip-compressed, detected by ".gz" in the name) and writes an
 * 8-bit grey PNG with one row per second of stream (per -s samples), W = -w pixels wide.  Same command line as the
 * reference's; no FFTW or libpng (-f is accepted and only checked).
 *
 * Pipeline: one group at fs with no clients and one band spectrum xlg_add_spectrum(W, fs / W, fs % W,
 * XLG_SPECTRUM_POWER), whose rows are the reference's (include/xlating_group.h).  The file is read into pinned
 * blocks submitted with XLG_INPUT_KEEP, so the next read overlaps the copy and the kernels; each ticket's rows are
 * collected in order.  The host forms 10 * log10f(v) in float as spectrogram.c:156-163 does, then the pixel as
 * png_util_set_data does, (int)(dB + 255) clamped to [0, 255]: the pixels are a function of the power rows alone.
 *
 * With -a (not the reference's) the spectrum is xlg_add_spectrum_any's at the same parameters: every -w up to 65536
 * (and up to fs), widths above 4096 that are not powers of two through the chirp-z stage.  The widths the tool
 * serves without -a give the same rows, so the same image, with it.
 *
 * Height: floor(samples / fs), samples being the whole complex samples of the file (its size, or the gzip trailer's
 * size field for .gz, as the reference does), counted in 64 bits (the reference's uint32_t count wraps at 2^32
 * samples).  Exactly the rows whose full period lies in the file.
 */
#include <errno.h>
#include <getopt.h>
#include <math.h>
#include <signal.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>
#include <zlib.h>

#include "png_gray.h"
#include "xlating_group.h"

#define BLOCK_SAMPLES (1u << 20) /* complex samples per submitted block */
#define N_BUFS XLG_SLOTS

static volatile sig_atomic_t stop = 0;

static void on_signal(int signum) {
  (void)signum;
  stop = 1;
}

static void usage(void) {
  printf("Usage:\n");
  printf("  -h  print help\n");
  printf("  -w <width> image width (default: 1024)\n");
  printf("  -s <sampling_rate> sampling rate (default: 48000)\n");
  printf("  -d <data_format> data format: cu8, cs16, cf32 (default: cu8)\n");
  printf("  -i <input_file> I/Q input file\n");
  printf("  -o <output_file> spectrogram output\n");
  printf("  -a  any width up to 65536 (not only up to 4096 or a power of two), through the chirp-z transform\n");
  printf("  -f <fftw_flags> supported values: FFTW_ESTIMATE, FFTW_MEASURE (accepted for compatibility; the transform "
         "runs on the GPU). Default: FFTW_MEASURE\n");
}

typedef struct {
  FILE *fp;
  gzFile gz;
} iq_in;

/* Reads up to `bytes`; returns the bytes read (fewer only at the end of the data or on an error). */
static size_t iq_read(iq_in *in, void *dst, size_t bytes) {
  if (in->fp != NULL) return fread(dst, 1, bytes, in->fp);
  size_t got = 0;
  while (got < bytes) {
    const unsigned ask = (unsigned)((bytes - got) > (1u << 30) ? (1u << 30) : (bytes - got));
    const int n = gzread(in->gz, (char *)dst + got, ask);
    if (n <= 0) break;
    got += (size_t)n;
  }
  return got;
}

int main(int argc, char **argv) {
  int width = 1024;
  double fs_arg = 48000;
  const char *data_format = "cu8", *input_file = NULL, *output_file = NULL, *fftw_flags = "FFTW_MEASURE";
  int opt, any_width = 0;
  while ((opt = getopt(argc, argv, "ahw:s:d:i:o:f:")) != -1) {
    switch (opt) {
      case 'a':
        any_width = 1;
        break;
      case 'h':
        usage();
        return EXIT_SUCCESS;
      case 'w':
        width = atoi(optarg);
        break;
      case 's':
        fs_arg = atof(optarg);
        break;
      case 'd':
        data_format = optarg;
        break;
      case 'i':
        input_file = optarg;
        break;
      case 'o':
        output_file = optarg;
        break;
      case 'f':
        fftw_flags = optarg;
        break;
      default:
        return EXIT_FAILURE;
    }
  }

  /* the reference's checks and messages (spectrogram.c:56-76); its rate is (uint32_t) atof(-s), which is defined
   * only for values in [0, 2^32): anything below 1 is its rate 0 */
  if (input_file == NULL) {
    fprintf(stderr, "-i (input file) parameter is missing\n");
    return EXIT_FAILURE;
  }
  if (output_file == NULL) {
    fprintf(stderr, "-o (output file) parameter is missing\n");
    return EXIT_FAILURE;
  }
  if (width <= 0) {
    fprintf(stderr, "-w (width) should be positive. got: %d\n", width);
    return EXIT_FAILURE;
  }
  if (!(fs_arg >= 1)) {
    fprintf(stderr, "-s (sampling_rate) should be positive. got: %d\n", 0);
    return EXIT_FAILURE;
  }
  /* the group's row period R = fs must stay below 2^31 */
  if (fs_arg >= 2147483648.0) {
    fprintf(stderr, "-s (sampling_rate) %.0f is too high: at most %u\n", fs_arg, 2147483647u);
    return EXIT_FAILURE;
  }
  const uint32_t fs = (uint32_t)fs_arg;
  if ((uint32_t)width > fs) {
    fprintf(stderr, "-w (%d) is too wide for sampling rate %u\n", width, fs);
    return EXIT_FAILURE;
  }
  const uint32_t W = (uint32_t)width;
  if (any_width && W > 65536) {
    fprintf(stderr, "-w (%d) is not served: widths up to 65536\n", width);
    return EXIT_FAILURE;
  }
  if (!any_width && (W > 65536 || (W > 4096 && (W & (W - 1)) != 0))) {
    fprintf(stderr, "-w (%d) is not served: widths up to 4096, or powers of two up to 65536\n", width);
    return EXIT_FAILURE;
  }
  int fmt;
  size_t sample_bytes;
  if (strcmp(data_format, "cu8") == 0) {
    fmt = XLG_FMT_CU8;
    sample_bytes = 2;
  } else if (strcmp(data_format, "cs16") == 0) {
    fmt = XLG_FMT_CS16;
    sample_bytes = 4;
  } else if (strcmp(data_format, "cf32") == 0) {
    fmt = XLG_FMT_CF32;
    sample_bytes = 8;
  } else {
    fprintf(stderr, "unsupported data format: %s\n", data_format);
    return EXIT_FAILURE;
  }

  /* the input and its length in complex samples (iq_file.c:35-80, 177-198) */
  iq_in in = {NULL, NULL};
  uint64_t samples = 0;
  if (strstr(input_file, ".gz") != NULL) {
    FILE *fp = fopen(input_file, "rb");
    if (fp == NULL) {
      fprintf(stderr, "unable to read input file %s: %s\n", input_file, strerror(errno));
      return EXIT_FAILURE;
    }
    unsigned char t[4];
    if (fseek(fp, -4, SEEK_END) != 0 || fread(t, 1, 4, fp) != 4) {
      fprintf(stderr, "premature end of file %s\n", input_file);
      fclose(fp);
      return EXIT_FAILURE;
    }
    fclose(fp);
    /* gzip's ISIZE: the uncompressed size mod 2^32 */
    const uint32_t isize = (uint32_t)t[0] | ((uint32_t)t[1] << 8) | ((uint32_t)t[2] << 16) | ((uint32_t)t[3] << 24);
    samples = isize / sample_bytes;
    in.gz = gzopen(input_file, "rb");
    if (in.gz == NULL) {
      fprintf(stderr, "unable to read input file %s: %s\n", input_file, strerror(errno));
      return EXIT_FAILURE;
    }
    gzbuffer(in.gz, 128 * 1024);
  } else {
    in.fp = fopen(input_file, "rb");
    if (in.fp == NULL) {
      fprintf(stderr, "unable to read input file %s: %s\n", input_file, strerror(errno));
      return EXIT_FAILURE;
    }
    if (fseeko(in.fp, 0, SEEK_END) != 0) {
      fprintf(stderr, "unable to read input file %s: %s\n", input_file, strerror(errno));
      fclose(in.fp);
      return EXIT_FAILURE;
    }
    const off_t size = ftello(in.fp);
    rewind(in.fp);
    samples = size > 0 ? (uint64_t)size / sample_bytes : 0;
  }
  const uint64_t height = samples / fs;
  int rc = EXIT_FAILURE;
  if (height == 0) {
    fprintf(stderr, "input file %s holds %llu samples, fewer than one row of %u\n", input_file,
            (unsigned long long)samples, fs);
    goto close_input;
  }
  if (height > 0x7fffffffu) {
    fprintf(stderr, "input file %s is too long: %llu rows\n", input_file, (unsigned long long)height);
    goto close_input;
  }
  if (strcmp(fftw_flags, "FFTW_MEASURE") != 0 && strcmp(fftw_flags, "FFTW_ESTIMATE") != 0)
    fprintf(stderr, "unsupported fftw flag: %s. Fallback to FFTW_ESTIMATE\n", fftw_flags);

  FILE *png_fp = fopen(output_file, "wb");
  if (png_fp == NULL) {
    fprintf(stderr, "unable to write to output: %s\n", output_file);
    goto close_input;
  }
  png_gray *png = NULL;
  float *db = malloc(sizeof(float) * W);
  uint8_t *pix = malloc(W);
  if (db == NULL || pix == NULL || png_gray_open(png_fp, W, (uint32_t)height, &png) != 0) {
    fprintf(stderr, "unable to initialize png\n");
    free(db);
    free(pix);
    fclose(png_fp);
    unlink(output_file);
    goto close_input;
  }

  struct sigaction sa;
  memset(&sa, 0, sizeof(sa));
  sa.sa_handler = on_signal;
  sigemptyset(&sa.sa_mask);
  sigaction(SIGINT, &sa, NULL);
  sigaction(SIGTERM, &sa, NULL);
  sigaction(SIGHUP, &sa, NULL);

  xlg_group *g = NULL;
  int sid = -1;
  void *bufs[N_BUFS] = {NULL};
  int64_t buf_ticket[N_BUFS];
  const uint64_t total = height * (uint64_t)fs; /* the samples the rows read, skips included */
  uint64_t sent = 0, rows_done = 0;
  int64_t next_read = 0, submitted = 0; /* tickets whose rows were written / tickets submitted */
  int failed = 0;
  int code = xlg_create(0, fs, 2 * BLOCK_SAMPLES, 0, &g);
  if (code == 0 && any_width) {
    const xlg_spectrum_desc desc = {W, fs / W, fs % W, XLG_SPECTRUM_POWER, 0, XLG_SPECTRUM_MAX, NULL};
    code = xlg_add_spectrum_any(g, XLG_SOURCE_BAND, 0, &desc, &sid);
  } else if (code == 0) {
    code = xlg_add_spectrum(g, W, fs / W, fs % W, XLG_SPECTRUM_POWER, &sid);
  }
  if (code != 0) {
    fprintf(stderr, "unable to start the GPU spectrum: %d\n", code);
    failed = 1;
  }
  for (int i = 0; i < N_BUFS && !failed; i++) {
    buf_ticket[i] = -1;
    bufs[i] = xlg_alloc_pinned(BLOCK_SAMPLES * sample_bytes);
    if (bufs[i] == NULL) {
      fprintf(stderr, "unable to allocate pinned input buffers\n");
      failed = 1;
    }
  }

  while (!failed && (sent < total || next_read < submitted)) {
    /* write the rows of the oldest ticket once XLG_SLOTS - 1 newer ones are in flight, or at the end */
    while (next_read < submitted && (submitted - next_read >= XLG_SLOTS - 1 || sent == total)) {
      const float *rows = NULL;
      size_t n_rows = 0;
      if (xlg_wait(g, next_read) != 0 || xlg_spectrum_output(g, next_read, sid, &rows, &n_rows) != 0) {
        fprintf(stderr, "the GPU spectrum failed\n");
        failed = 1;
        break;
      }
      for (size_t r = 0; r < n_rows && rows_done < height; r++, rows_done++) {
        const float *v = rows + r * W;
        for (uint32_t j = 0; j < W; j++) db[j] = 10 * log10f(v[j]);
        for (uint32_t j = 0; j < W; j++) {
          int pixel = (int)(db[j] + 255);
          pix[j] = (uint8_t)(pixel > 255 ? 255 : pixel < 0 ? 0 : pixel);
        }
        if (png_gray_row(png, pix) != 0) {
          fprintf(stderr, "unable to write to output: %s\n", output_file);
          failed = 1;
          break;
        }
      }
      next_read++;
      if (failed) break;
    }
    if (failed || stop) break;
    if (sent == total) continue;
    const int i = (int)(submitted % N_BUFS);
    if (buf_ticket[i] >= 0 && xlg_input_consumed(g, buf_ticket[i]) != 0) {
      fprintf(stderr, "the GPU spectrum failed\n");
      failed = 1;
      break;
    }
    const uint64_t want = total - sent < BLOCK_SAMPLES ? total - sent : BLOCK_SAMPLES;
    const size_t bytes = (size_t)want * sample_bytes;
    if (iq_read(&in, bufs[i], bytes) != bytes) {
      fprintf(stderr, "premature end of file %s: %llu of %llu samples read\n", input_file,
              (unsigned long long)sent, (unsigned long long)total);
      failed = 1;
      break;
    }
    const int64_t t = xlg_submit(g, fmt, bufs[i], 2 * (size_t)want, XLG_INPUT_KEEP);
    if (t < 0) {
      fprintf(stderr, "the GPU spectrum refused a block: %lld\n", (long long)t);
      failed = 1;
      break;
    }
    buf_ticket[i] = t;
    submitted = t + 1;
    sent += want;
  }
  if (stop) fprintf(stderr, "Signal caught, exiting!\n");

  /* drain: the group reads the pinned buffers until its tickets complete */
  if (g != NULL && submitted > 0) xlg_wait(g, submitted - 1);
  if (g != NULL) xlg_destroy(g);
  for (int i = 0; i < N_BUFS; i++)
    if (bufs[i] != NULL) xlg_free_pinned(bufs[i]);
  free(db);
  free(pix);
  if (!failed && !stop && rows_done != height) {
    fprintf(stderr, "the GPU spectrum returned %llu of %llu rows\n", (unsigned long long)rows_done,
            (unsigned long long)height);
    failed = 1;
  }
  if (failed || stop) {
    png_gray_free(png);
    fclose(png_fp);
    unlink(output_file); /* no partial image is left that looks complete */
  } else if (png_gray_finish(png) != 0 || fclose(png_fp) != 0) {
    fprintf(stderr, "unable to write to output: %s\n", output_file);
    unlink(output_file);
  } else {
    rc = EXIT_SUCCESS;
  }

close_input:
  if (in.fp != NULL) fclose(in.fp);
  if (in.gz != NULL) gzclose(in.gz);
  return rc;
}
