/*
 * oracle/pn2_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * CPU restatement of the four PointNet++ native ops that SAM-6D's Pose
 * Estimation Model calls at inference.  The reference implements them only as
 * CUDA kernels (every host wrapper ends in TORCH_CHECK(false, "CPU not
 * supported")), so this file restates the *algorithm* of each kernel in plain
 * C, including the floating-point expression order the reference compiles to
 * (nvcc -fmad=true contracts  a*a + b*b + c*c  into  fma(c,c, fma(b,b, a*a));
 * the contraction nvcc applies to the reference kernel: FMUL, FFMA, FFMA).
 *
 * Reference (paths relative to SAM-6D/Pose_Estimation_Model/model/pointnet2):
 *   fps          : _ext_src/src/sampling_gpu.cu:75-178  (+ host temp init 1e10, sampling.cpp:78-80)
 *   gather       : _ext_src/src/sampling_gpu.cu:13-25
 *   ball_query   : _ext_src/src/ball_query_gpu.cu:14-49 (output pre-zeroed, ball_query.cpp:24-26)
 *   group_points : _ext_src/src/group_points_gpu.cu:13-33
 *   block size   : _ext_src/include/cuda_utils.h:20-24  (opt_n_threads)
 *
 * Parity status: pinned on the GPU box against the reference's own CUDA
 * kernels when oracle/_ref/ holds the reference extension (tests/test_gpu_pn2.py);
 * otherwise pinned only through the golden vectors under tests/golden/.
 *
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC (see oracle/Makefile).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* cuda_utils.h:20-24 -- min(2^floor(log2 n), 512), at least 1 */
static int opt_n_threads(int work_size) {
  int pow_2 = (int)(log((double)work_size) / log(2.0));
  int t = 1 << pow_2;
  if (t > 512) t = 512;
  if (t < 1) t = 1;
  return t;
}

int pn2_oracle_block_size(int n) { return opt_n_threads(n); }

static inline float sqdist_ref(float x1, float y1, float z1, float x2, float y2, float z2) {
  /* (x2-x1)*(x2-x1) + (y2-y1)*(y2-y1) + (z2-z1)*(z2-z1) with nvcc's contraction */
  float dx = x2 - x1, dy = y2 - y1, dz = z2 - z1;
  float d = dx * dx;
  d = fmaf(dy, dy, d);
  d = fmaf(dz, dz, d);
  return d;
}

/*
 * Furthest point sampling.  xyz (b,n,3) f32 -> idx (b,m) i32.
 * The reference runs one CTA of `bs` threads per cloud: thread t scans
 * k = t, t+bs, ... keeping (best, besti) under a strict '>' (first k wins a
 * tie inside a thread), then a shared-memory tree reduce where slot t absorbs
 * slot t+s only if strictly greater (slot t wins a tie).  Net effect on exact
 * ties: the smallest BIT-REVERSED (k mod bs) wins, then the smallest k.  We emulate
 * the threads and the tree literally.
 */
void pn2_oracle_fps(const float *xyz, int b, int n, int m, int32_t *idx) {
  if (m <= 0) return;
  int bs = opt_n_threads(n);
  float *temp = (float *)malloc(sizeof(float) * (size_t)n);
  float *best = (float *)malloc(sizeof(float) * (size_t)bs);
  int *besti = (int *)malloc(sizeof(int) * (size_t)bs);
  for (int bi = 0; bi < b; ++bi) {
    const float *p = xyz + (size_t)bi * n * 3;
    int32_t *out = idx + (size_t)bi * m;
    for (int k = 0; k < n; ++k) temp[k] = 1e10f;
    int old = 0;
    out[0] = 0;
    for (int j = 1; j < m; ++j) {
      float x1 = p[old * 3 + 0], y1 = p[old * 3 + 1], z1 = p[old * 3 + 2];
      for (int t = 0; t < bs; ++t) { best[t] = -1.f; besti[t] = 0; }
      for (int k = 0; k < n; ++k) {
        int t = k % bs;
        float d = sqdist_ref(x1, y1, z1, p[k * 3 + 0], p[k * 3 + 1], p[k * 3 + 2]);
        float d2 = fminf(d, temp[k]);
        temp[k] = d2;
        if (d2 > best[t]) { best[t] = d2; besti[t] = k; }
      }
      for (int s = bs / 2; s >= 1; s >>= 1) {
        for (int t = 0; t < s; ++t) {
          float v1 = best[t], v2 = best[t + s];
          if (v2 > v1) { best[t] = v2; besti[t] = besti[t + s]; }
        }
      }
      old = besti[0];
      out[j] = old;
    }
  }
  free(temp); free(best); free(besti);
}

/* gather: points (b,c,n), idx (b,m) -> out (b,c,m) */
void pn2_oracle_gather(const float *points, const int32_t *idx, int b, int c, int n, int m, float *out) {
  for (int i = 0; i < b; ++i)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < m; ++j)
        out[((size_t)i * c + l) * m + j] = points[((size_t)i * c + l) * n + idx[(size_t)i * m + j]];
}

/*
 * ball query: new_xyz (b,m,3), xyz (b,n,3) -> idx (b,m,nsample), zero-filled
 * first; first `nsample` hits with d2 < r*r in ascending k; on the first hit
 * every slot is set to that k.
 */
void pn2_oracle_ball_query(const float *new_xyz, const float *xyz, int b, int n, int m, float radius,
                           int nsample, int32_t *idx) {
  float radius2 = radius * radius;
  memset(idx, 0, sizeof(int32_t) * (size_t)b * m * nsample);
  for (int bi = 0; bi < b; ++bi) {
    const float *q = new_xyz + (size_t)bi * m * 3;
    const float *p = xyz + (size_t)bi * n * 3;
    int32_t *o = idx + (size_t)bi * m * nsample;
    for (int j = 0; j < m; ++j) {
      float nx = q[j * 3 + 0], ny = q[j * 3 + 1], nz = q[j * 3 + 2];
      int cnt = 0;
      for (int k = 0; k < n && cnt < nsample; ++k) {
        /* (new_x - x)^2 + (new_y - y)^2 + (new_z - z)^2, contracted like nvcc */
        float dx = nx - p[k * 3 + 0], dy = ny - p[k * 3 + 1], dz = nz - p[k * 3 + 2];
        float d2 = dx * dx;
        d2 = fmaf(dy, dy, d2);
        d2 = fmaf(dz, dz, d2);
        if (d2 < radius2) {
          if (cnt == 0)
            for (int l = 0; l < nsample; ++l) o[(size_t)j * nsample + l] = k;
          o[(size_t)j * nsample + cnt] = k;
          ++cnt;
        }
      }
    }
  }
}

/* group: points (b,c,n), idx (b,np,ns) -> out (b,c,np,ns) */
void pn2_oracle_group(const float *points, const int32_t *idx, int b, int c, int n, int np, int ns,
                      float *out) {
  for (int bi = 0; bi < b; ++bi)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < np; ++j)
        for (int k = 0; k < ns; ++k) {
          int ii = idx[((size_t)bi * np + j) * ns + k];
          out[(((size_t)bi * c + l) * np + j) * ns + k] = points[((size_t)bi * c + l) * n + ii];
        }
}
