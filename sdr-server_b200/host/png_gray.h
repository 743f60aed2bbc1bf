/*
 * host/png_gray.h -- a streaming writer of 8-bit grey PNG images on zlib alone: IHDR, IDAT chunks written as rows
 * arrive, IEND; no interlace, filter type 0 on every row, CRCs from zlib's crc32.  The spectrogram tool's images
 * are this format (the reference writes them through libpng; the decoded pixels are the same, the bytes need not be).
 */
#ifndef XLATING_B200_PNG_GRAY_H_
#define XLATING_B200_PNG_GRAY_H_

#include <stdint.h>
#include <stdio.h>

typedef struct png_gray png_gray;

/* Starts an image of width x height pixels on fp (kept open; the caller closes it) and writes the signature and
 * IHDR.  0, or -EINVAL for a zero or too large (> 2^31 - 1) dimension, -ENOMEM, -EIO on a write error. */
int png_gray_open(FILE *fp, uint32_t width, uint32_t height, png_gray **out);
/* Appends one row of `width` pixels.  -EINVAL after `height` rows, -EIO on a write error. */
int png_gray_row(png_gray *p, const uint8_t *row);
/* Ends the image: the last IDAT chunks and IEND.  -EINVAL unless exactly `height` rows were written, -EIO on a write
 * error; the file is a valid PNG only when this returns 0.  Frees p either way. */
int png_gray_finish(png_gray *p);
/* Frees an unfinished image without ending it. */
void png_gray_free(png_gray *p);

#endif /* XLATING_B200_PNG_GRAY_H_ */
