/* tests/png_gray_shim.c -- drives sdr-server_b200/host/png_gray.c from Python: writes height rows of width pixels
 * (row-major) to path, one png_gray_row per row.  Returns png_gray's code, or -1 if the file cannot be opened. */
#include <stdio.h>

#include "png_gray.h"

int png_gray_write_file(const char *path, uint32_t width, uint32_t height, const uint8_t *pixels) {
  FILE *fp = fopen(path, "wb");
  if (fp == NULL) return -1;
  png_gray *p = NULL;
  int rc = png_gray_open(fp, width, height, &p);
  for (uint32_t r = 0; rc == 0 && r < height; r++) rc = png_gray_row(p, pixels + (size_t)r * width);
  if (rc == 0)
    rc = png_gray_finish(p);
  else
    png_gray_free(p);
  fclose(fp);
  return rc;
}

/* A row past the announced height, then finish: both must fail. */
int png_gray_overrun(const char *path) {
  FILE *fp = fopen(path, "wb");
  if (fp == NULL) return -1;
  png_gray *p = NULL;
  const uint8_t row[2] = {1, 2};
  int rc = png_gray_open(fp, 2, 1, &p);
  if (rc == 0) rc = png_gray_row(p, row);
  const int extra = rc == 0 ? png_gray_row(p, row) : 0;
  png_gray_free(p);
  fclose(fp);
  return rc == 0 && extra != 0 ? 0 : 1;
}

/* finish with fewer rows than announced must fail */
int png_gray_short(const char *path) {
  FILE *fp = fopen(path, "wb");
  if (fp == NULL) return -1;
  png_gray *p = NULL;
  const uint8_t row[2] = {1, 2};
  int rc = png_gray_open(fp, 2, 3, &p);
  if (rc == 0) rc = png_gray_row(p, row);
  const int fin = rc == 0 ? png_gray_finish(p) : 0;
  fclose(fp);
  return rc == 0 && fin != 0 ? 0 : 1;
}
