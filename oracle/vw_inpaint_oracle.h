/* vw_inpaint_oracle.h -- CPU oracle of fill_holes_grass (src/vw/Image/InpaintView.h:239-311), written loop for loop from
 * the reference (test infrastructure only).  For an output window (x0, y0, ow, oh) inside a w x h disparity:
 *   1. tile     = bbox.expand(len) cropped to the image (FillHolesGrass::prerasterize, :266-279)
 *   2. holes    = 8-connected components of the tile's invalid pixels (BlobIndexThreaded with one task, BlobIndex.h:113-305);
 *                 a hole goes when its pixel count is > len*len (len*len > 0, :445-453) or when its half-open bounding box
 *                 is wider or taller than len (wipe_big_blobs, :457-477)
 *   3. skip     = a hole whose bbox.expand(1) has min < 0 or max >= tile cols / rows (InpaintTask, InpaintView.h:76-80)
 *   4. order    = grassfire distance of the hole inside bbox.expand(1) (Grassfire.h:79-170), d = 1..max, column-major
 *   5. inpaint  = 10 * max^2 in-place sweeps of the 8-neighbour stencil (.176765 corners, .073235 edges, :114-135): each
 *                 product in double, each += narrowed to float, the store converts to the pixel type (int32 truncates)
 *   6. output   = the window of the tile, filled pixels valid (1), every other pixel copied
 * Pixels are {dx, dy, valid} triples of int32 (type 0, PixelMask<Vector2i>) or float (type 1, PixelMask<Vector2f>), dense
 * row-major.  Built with the reference's -O3 -msse4.1 -ffp-contract=off. */
#ifndef VW_INPAINT_ORACLE_H
#define VW_INPAINT_ORACLE_H

/* stats (may be NULL): [0] holes found in the tile, [1] holes filled, [2] the largest 10 * max_distance^2 of a filled hole.
 * Returns 0, or -1 for a window outside the image or a negative len. */
int vwi_fill_holes_grass(int type, const void* in, int w, int h, int len, int x0, int y0, int ow, int oh, void* out, int* stats);

#endif
