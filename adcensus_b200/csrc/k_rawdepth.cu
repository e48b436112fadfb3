// k_rawdepth.cu -- the high-bit-depth instantiations of the view ingestion kernel k_view_ingest (k_image.cuh), one per
// format x source geometry: five containers (16-bit words holding 10, 12 or 16 significant bits; the PFNC 10p and 12p
// bit streams) x mono and the four Bayer patterns, all reading through rd_sample, the mosaics through mosaic_px.  Container, depth and pattern are template constants, so
// the shift of the depth reduction and the field width of the packed readers are immediates and the kernels take the
// arguments every other format takes.
//
// Plain ingestion: each thread converts four consecutive output pixels; a mono pixel is one sample (one 16-bit load, or
// two byte loads for a packed field), a Bayer pixel nine samples from the clamped 3x3 neighbourhood, demosaiced at full
// depth and then reduced to 8 bits.  Neighbouring lanes take neighbouring pixels, so a warp's loads cover contiguous
// stretches of three rows and L1 serves the reuse.  Rectified ingestion: a 4x4 window of samples per output pixel where
// no clamp applies, neighbour by neighbour at the frame's edges; a neighbour outside the frame is 0.  No shared memory:
// see DESIGN.md section 19.
#include "k_image.cuh"

ADC_IMG_RAWDEPTH_FORMATS(II_VIEWS)
