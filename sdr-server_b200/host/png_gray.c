/*
 * host/png_gray.c -- see png_gray.h.  Chunk layout (PNG specification, 5.3): a 4-byte big-endian length, the
 * 4-byte type, the data, and the CRC-32 of type and data.
 */
#include "png_gray.h"

#include <errno.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

#define PNG_GRAY_IDAT 65536 /* bytes of compressed data per IDAT chunk */

struct png_gray {
  FILE *fp;
  uint32_t width, height, rows;
  z_stream z;
  unsigned char *line; /* filter byte + one row */
  unsigned char out[PNG_GRAY_IDAT];
};

static void be32(unsigned char *b, uint32_t v) {
  b[0] = (unsigned char)(v >> 24);
  b[1] = (unsigned char)(v >> 16);
  b[2] = (unsigned char)(v >> 8);
  b[3] = (unsigned char)v;
}

static int chunk(FILE *fp, const char *type, const unsigned char *data, uint32_t len) {
  unsigned char head[8], crc[4];
  be32(head, len);
  memcpy(head + 4, type, 4);
  uLong c = crc32(0L, Z_NULL, 0);
  c = crc32(c, head + 4, 4);
  if (len > 0) c = crc32(c, data, len);
  be32(crc, (uint32_t)c);
  if (fwrite(head, 1, 8, fp) != 8 || (len > 0 && fwrite(data, 1, len, fp) != len) || fwrite(crc, 1, 4, fp) != 4)
    return -EIO;
  return 0;
}

/* Runs deflate with `flush` and writes every full output buffer (and, for Z_FINISH, the rest) as an IDAT chunk. */
static int pump(png_gray *p, int flush) {
  for (;;) {
    const int rc = deflate(&p->z, flush);
    if (rc == Z_STREAM_ERROR) return -EIO;
    const uint32_t have = (uint32_t)(PNG_GRAY_IDAT - p->z.avail_out);
    if (p->z.avail_out == 0 || (flush == Z_FINISH && have > 0)) {
      if (chunk(p->fp, "IDAT", p->out, have)) return -EIO;
      p->z.next_out = p->out;
      p->z.avail_out = PNG_GRAY_IDAT;
    }
    if (flush == Z_FINISH ? rc == Z_STREAM_END : p->z.avail_in == 0 && p->z.avail_out > 0) return 0;
  }
}

int png_gray_open(FILE *fp, uint32_t width, uint32_t height, png_gray **out) {
  *out = NULL;
  if (width == 0 || height == 0 || width > 0x7fffffffu || height > 0x7fffffffu) return -EINVAL;
  png_gray *p = calloc(1, sizeof(png_gray));
  if (p == NULL) return -ENOMEM;
  p->line = malloc((size_t)width + 1);
  if (p->line == NULL || deflateInit(&p->z, Z_DEFAULT_COMPRESSION) != Z_OK) {
    free(p->line);
    free(p);
    return -ENOMEM;
  }
  p->fp = fp;
  p->width = width;
  p->height = height;
  p->z.next_out = p->out;
  p->z.avail_out = PNG_GRAY_IDAT;
  static const unsigned char sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  unsigned char ihdr[13];
  be32(ihdr, width);
  be32(ihdr + 4, height);
  ihdr[8] = 8;   /* bit depth */
  ihdr[9] = 0;   /* colour type: grey */
  ihdr[10] = 0;  /* compression: deflate */
  ihdr[11] = 0;  /* filter method 0 */
  ihdr[12] = 0;  /* no interlace */
  if (fwrite(sig, 1, 8, fp) != 8 || chunk(fp, "IHDR", ihdr, 13)) {
    png_gray_free(p);
    return -EIO;
  }
  *out = p;
  return 0;
}

int png_gray_row(png_gray *p, const uint8_t *row) {
  if (p->rows >= p->height) return -EINVAL;
  p->line[0] = 0; /* filter type 0: none */
  memcpy(p->line + 1, row, p->width);
  p->z.next_in = p->line;
  p->z.avail_in = p->width + 1;
  if (pump(p, Z_NO_FLUSH)) return -EIO;
  p->rows++;
  return 0;
}

int png_gray_finish(png_gray *p) {
  int rc = p->rows == p->height ? 0 : -EINVAL;
  if (rc == 0) {
    p->z.next_in = NULL;
    p->z.avail_in = 0;
    if (pump(p, Z_FINISH) || chunk(p->fp, "IEND", NULL, 0) || fflush(p->fp) != 0) rc = -EIO;
  }
  png_gray_free(p);
  return rc;
}

void png_gray_free(png_gray *p) {
  if (p == NULL) return;
  deflateEnd(&p->z);
  free(p->line);
  free(p);
}
