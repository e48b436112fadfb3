// k_bayer.cu -- the Bayer-mosaic instantiations of the view ingestion kernel k_view_ingest (k_image.cuh): one per
// pattern x source geometry, all reading through mosaic_px.
//
// Plain ingestion: each thread demosaics four consecutive output pixels, nine byte loads each from the clamped 3x3
// neighbourhood; neighbouring lanes take neighbouring pixels, so a warp's loads hit the same three stretches of rows and
// L1 serves the 9x reuse.  Rectified ingestion: each of the four bilinear neighbours inside the frame is demosaiced the
// same way (a 4x4 raw window per output pixel), a neighbour outside the frame is 0; a 2 x 2 AREA block away from the
// frame's edges likewise takes its four sites from one 4x4 window.  A frame narrower or lower than 3
// pixels gives all-zero views without a load.  No shared memory: see DESIGN.md section 17 for the measurements.
#include "k_image.cuh"

ADC_IMG_BAYER_FORMATS(II_VIEWS)
