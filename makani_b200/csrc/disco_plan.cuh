// The device plan of the DISCO convolution (disco.cu), shared with the neighbourhood attention kernels (attention.cu), which read its support
// lists: both orderings, the band tables and the per-point values.
#pragma once
#include "common.cuh"

namespace b200sht {

struct DiscoPlan {
  int nlat_in, nlon_in, nlat_out, nlon_out, K, Kp, pscale;
  long long nnz, npts;
  int* d_fwd_rowptr;   // [nlat_out][nlat_in + 1] first point of (t, row >= i)
  int2* d_fwd_band;    // [nlat_out] rows [lo, hi) of the input band of t
  int2* d_fwd_pos;     // [npts] (i, j)
  float* d_fwd_val;    // [npts][Kp]
  int* d_adj_rowptr;   // [nlat_in][nlat_out + 1] first point of (i, t' >= t)
  int2* d_adj_band;    // [nlat_in] output rows [lo, hi) that reach i
  int2* d_adj_pos;     // [npts] (t, j)
  float* d_adj_val;    // [npts][Kp]
  size_t bytes;
};

}  // namespace b200sht

struct b200sht_disco_plan : public b200sht::DiscoPlan {};
