// lsdreg.cu — unity translation unit of liblsdreg.so (device functions and __constant__ tables are
// shared between kernels without relocatable device code).
#include "map.cu"
#include "voxelgrid.cu"
#include "lio.cu"
#include "reg.cu"
#include "loop.cu"
#include "vfe.cu"
#include "imu.cu"
#include "filters.cu"
#include "localmap.cu"
#include "keyframe_io.cu"
#include "scancontext.cu"
#include "fastlio_seam.cu"
