// Marching cubes over a dense SDF grid: deterministic, scan-based, shared vertices
// (SURVEY.md rows a22 / K3-K6).
//
// Semantics follow MCGpu/CudaKernels.cu:304-521 of the reference:
//   * cube index bit c set iff sdf[corner c] < iso; classic 256-case table;
//   * a vertex exists once per crossed grid edge and is owned by the voxel whose min
//     corner starts the edge (edges 0 / 3 / 8 = x / y / z), only if that voxel is a valid
//     cell (i<nx-1, j<ny-1, k<nz-1); faces that reference an edge owned by a boundary-layer
//     voxel get index -1 (the reference leaves edge_point_state at -1 there);
//   * t = (float)((double)(iso-v1)/(double)(v2-v1)), 0.5 when v1==v2 (d_fGetOffset,
//     CudaKernels.cu:304-313); edge 3 runs from corner 3 to corner 0, i.e. y = j + (1 - t);
//   * world position = fmaf(pos, step, min) (d_scale_vertices, :513-521);
//   * face winding reversed (d_conver_ijkd_to_pindex, :492-505).
// The reference numbers vertices/faces with atomicAdd (order = race winner), fills a
// 12 B/voxel state volume with -1 on every call, and writes/reads 48 B of (i,j,k,dir) keys
// per face.  Here the order is canonical and no per-voxel state volume exists:
//
//   pass 1 (classify): one warp per 32-voxel word along k. Ballots give three bit-planes
//       (which owned x/y/z edges are crossed), a warp sum gives #triangles.  Per word:
//       20 B (0.625 B/voxel).  Each CTA owns a contiguous chunk of words and writes
//       CTA-local exclusive prefixes plus one CTA total.
//   scan: one tiny single-CTA kernel over the CTA totals (<= 18k entries at 513^3).
//   pass 2 (emit): words with no vertex and no face exit after reading their 20 B; active
//       words re-read their 4x33 SDF values (L2 resident) and write vertices / faces
//       straight to their final slots.  A vertex id is
//          cta_base + word_prefix + popc(planes below k) (+ lower dirs at k),
//       so neighbours' ids are found by address arithmetic, not through a state volume.
//
// HBM traffic: 4 B/voxel (grid, once from DRAM; the re-read of active words hits L2)
// + 1.25 B/voxel (word info write + read) + 12 B/vertex + 24 B/face.
#include "common.cuh"

namespace {

// Public-domain Lorensen-Cline / Bourke / Bloyd triangulation, one case per 64-bit word,
// 4 bits per edge id, 0xF terminated.  Content is necessarily identical to
// a2iTriangleConnectionTable (MCGpu/CudaKernels.cu:37-298): face parity depends on it.
// The 256-entry edge-flag table of the reference is not stored: edge e is crossed iff
// its two end corners differ in the cube index (asserted for all 256 cases in
// tests/test_mc_tables.py).
__device__ __constant__ uint64_t kTriPacked[256] = {
    0xffffffffffffffffULL, 0xfffffffffffff380ULL, 0xfffffffffffff910ULL, 0xffffffffff189381ULL,
    0xfffffffffffffa21ULL, 0xffffffffffa21380ULL, 0xffffffffff920a29ULL, 0xfffffff89a8a2382ULL,
    0xfffffffffffff2b3ULL, 0xffffffffff0b82b0ULL, 0xffffffffffb32091ULL, 0xfffffffb89b912b1ULL,
    0xffffffffff3ab1a3ULL, 0xfffffffab8a801a0ULL, 0xfffffff9ab9b3093ULL, 0xffffffffffb8aa89ULL,
    0xfffffffffffff874ULL, 0xffffffffff437034ULL, 0xffffffffff748910ULL, 0xfffffff137174914ULL,
    0xffffffffff748a21ULL, 0xfffffffa21403743ULL, 0xfffffff748209a29ULL, 0xffff4973727929a2ULL,
    0xffffffffff2b3748ULL, 0xfffffff40242b74bULL, 0xfffffffb32748109ULL, 0xffff1292b9b49b74ULL,
    0xfffffff487ab31a3ULL, 0xffff4b7401b41ab1ULL, 0xffff30bab9b09874ULL, 0xfffffffab99b4b74ULL,
    0xfffffffffffff459ULL, 0xffffffffff380459ULL, 0xffffffffff051450ULL, 0xfffffff513538458ULL,
    0xffffffffff459a21ULL, 0xfffffff594a21803ULL, 0xfffffff204245a25ULL, 0xffff8434535235a2ULL,
    0xffffffffffb32459ULL, 0xfffffff594b802b0ULL, 0xfffffffb32510450ULL, 0xffff584b82852512ULL,
    0xfffffff45931ab3aULL, 0xffffab81a8180594ULL, 0xffff30bab5b05045ULL, 0xfffffffb8aa85845ULL,
    0xffffffffff975879ULL, 0xfffffff375359039ULL, 0xfffffff751710870ULL, 0xffffffffff753351ULL,
    0xfffffff21a759879ULL, 0xffff37503505921aULL, 0xffff25a758528208ULL, 0xfffffff7533525a2ULL,
    0xfffffff2b3987597ULL, 0xffffb72029279759ULL, 0xffff751871810b32ULL, 0xfffffff51771b12bULL,
    0xffffb3a31a758859ULL, 0xf0aba010b7905075ULL, 0xf07570805a30b0abULL, 0xffffffffff5b75abULL,
    0xfffffffffffff56aULL, 0xffffffffff6a5380ULL, 0xffffffffff6a5109ULL, 0xfffffff6a5891381ULL,
    0xffffffffff162561ULL, 0xfffffff803621561ULL, 0xfffffff620609569ULL, 0xffff823625285895ULL,
    0xffffffffff56ab32ULL, 0xfffffff56a02b80bULL, 0xfffffff6a5b32910ULL, 0xffffb892b92916a5ULL,
    0xfffffff315356b36ULL, 0xffff6b51505b0b80ULL, 0xffff9505606306b3ULL, 0xfffffff89bb96956ULL,
    0xffffffffff8746a5ULL, 0xfffffffa56374034ULL, 0xfffffff7486a5091ULL, 0xffff49737179156aULL,
    0xfffffff874156216ULL, 0xffff743403625521ULL, 0xffff620560509748ULL, 0xf962695923497937ULL,
    0xfffffff56a4872b3ULL, 0xffffb720242746a5ULL, 0xffff6a5b32874910ULL, 0xf6a54b7b492b9129ULL,
    0xffff6b51535b3748ULL, 0xfb404b7b016b5b15ULL, 0xf74836b630560950ULL, 0xffff9b7974b96956ULL,
    0xffffffffffa4694aULL, 0xfffffff380a946a4ULL, 0xfffffff04606a10aULL, 0xffffa16468618138ULL,
    0xfffffff462421941ULL, 0xffff462942921803ULL, 0xffffffffff624420ULL, 0xfffffff624428238ULL,
    0xfffffff32b46a94aULL, 0xffff6a4a94b82280ULL, 0xffffa164606102b3ULL, 0xf1b8b12184a16146ULL,
    0xffff36b319639469ULL, 0xf14641916b0181b8ULL, 0xfffffff4600636b3ULL, 0xffffffffff86b846ULL,
    0xfffffffa98a876a7ULL, 0xffffa76a907a0370ULL, 0xffff0818717a176aULL, 0xfffffff37117a76aULL,
    0xffff768981861621ULL, 0xf937390976192962ULL, 0xfffffff206607087ULL, 0xffffffffff276237ULL,
    0xffff76898a86ab32ULL, 0xf7a9a76790b72702ULL, 0xfb32a767a1871081ULL, 0xffff17616a71b12bULL,
    0xf63136b619768698ULL, 0xffffffffff76b190ULL, 0xffff06b0b3607087ULL, 0xfffffffffffff6b7ULL,
    0xfffffffffffffb67ULL, 0xffffffffff67b803ULL, 0xffffffffff67b910ULL, 0xfffffff67b138918ULL,
    0xffffffffff7b621aULL, 0xfffffff7b6803a21ULL, 0xfffffff7b69a2092ULL, 0xffff89a38a3a27b6ULL,
    0xffffffffff726327ULL, 0xfffffff026067807ULL, 0xfffffff910732672ULL, 0xffff678891681261ULL,
    0xfffffff73171a67aULL, 0xffff801781a7167aULL, 0xffff7a69a0a70730ULL, 0xfffffff9a88a7a67ULL,
    0xffffffffff68b486ULL, 0xfffffff640603b63ULL, 0xfffffff109648b68ULL, 0xffff63b139369649ULL,
    0xfffffff1a28b6486ULL, 0xffff640b60b03a21ULL, 0xffff9a2920b648b4ULL, 0xf36463b34923a39aULL,
    0xfffffff264248328ULL, 0xffffffffff264240ULL, 0xffff834642432091ULL, 0xfffffff642241491ULL,
    0xffff1a6648168318ULL, 0xfffffff40660a01aULL, 0xf39a9303a6834364ULL, 0xffffffffff4a649aULL,
    0xffffffffffb67594ULL, 0xfffffff67b594380ULL, 0xfffffffb67045105ULL, 0xffff51345343867bULL,
    0xfffffffb6721a459ULL, 0xffff594380a217b6ULL, 0xffff204a24a45b67ULL, 0xf67b25a523453843ULL,
    0xfffffff945267327ULL, 0xffff786260680459ULL, 0xffff045051673263ULL, 0xf851584812786826ULL,
    0xffff73167161a459ULL, 0xf459078701671a61ULL, 0xfa737a6a305a4a04ULL, 0xffffa84a458a7a67ULL,
    0xfffffff98b9b6596ULL, 0xffff590650360b63ULL, 0xffffb65510b508b0ULL, 0xfffffff1355363b6ULL,
    0xffff65b8b9b59a21ULL, 0xfa21965690b603b0ULL, 0xf52025a50865b58bULL, 0xffff35a3a25363b6ULL,
    0xffff283265825985ULL, 0xfffffff260069659ULL, 0xf826283865081851ULL, 0xffffffffff612651ULL,
    0xf698965683a61631ULL, 0xffff06505960a01aULL, 0xffffffffffa65830ULL, 0xfffffffffffff65aULL,
    0xffffffffffb57a5bULL, 0xfffffff03857ba5bULL, 0xfffffff091ba57b5ULL, 0xffff1381897ba57aULL,
    0xfffffff15717b21bULL, 0xffffb27571721380ULL, 0xffff7b2209729579ULL, 0xf289823295b27257ULL,
    0xfffffff573532a52ULL, 0xffff52a578258028ULL, 0xffff2a37353a5109ULL, 0xf25752a278129289ULL,
    0xffffffffff573531ULL, 0xfffffff571170780ULL, 0xfffffff735539309ULL, 0xffffffffff795789ULL,
    0xfffffff8ba8a5485ULL, 0xffff03bba50b5405ULL, 0xffff54aba8a48910ULL, 0xf41314943b54a4baULL,
    0xffff8548b2582152ULL, 0xfb151b2b543b0b40ULL, 0xf58b8545b2950520ULL, 0xffffffffff3b2549ULL,
    0xffff483543253a52ULL, 0xfffffff0244252a5ULL, 0xf910854583a532a3ULL, 0xffff2492914252a5ULL,
    0xfffffff153358548ULL, 0xffffffffff501540ULL, 0xffff530509358548ULL, 0xfffffffffffff549ULL,
    0xfffffffba9b947b4ULL, 0xffffba97b9794380ULL, 0xffffb470414b1ba1ULL, 0xf4bab474a1843413ULL,
    0xffff219b294b97b4ULL, 0xf3801b2b197b9479ULL, 0xfffffff04224b47bULL, 0xffff42343824b47bULL,
    0xffff947732972a92ULL, 0xf70207872a4797a9ULL, 0xfa040a1a472a3a73ULL, 0xffffffffff4782a1ULL,
    0xfffffff317714194ULL, 0xffff178180714194ULL, 0xffffffffff347304ULL, 0xfffffffffffff784ULL,
    0xffffffffff8ba8a9ULL, 0xfffffffa9bb93903ULL, 0xfffffffba88a0a10ULL, 0xffffffffffa3ba13ULL,
    0xfffffff8b99b1b21ULL, 0xffff9b2921b93903ULL, 0xffffffffffb08b20ULL, 0xfffffffffffffb23ULL,
    0xfffffff98aa82832ULL, 0xffffffffff2902a9ULL, 0xffff8a1810a82832ULL, 0xfffffffffffff2a1ULL,
    0xffffffffff819831ULL, 0xfffffffffffff190ULL, 0xfffffffffffff830ULL, 0xffffffffffffffffULL,
};

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kWordsPerWarp = 32;
constexpr int kWordsPerCta = kWarps * kWordsPerWarp;  // 256 words = 8192 voxels
constexpr uint32_t kHasTris = 0x80000000u;

struct McLayout {
  int nx, ny, nz, nwz;
  long long nwords;
  int nctas;
  uint32_t *fx, *fy, *fz, *vpre, *tpre;  // [nwords]
  uint32_t* sgn;                         // [nwords] bit k of word (i,j,k/32): sdf[i,j,k] < iso
  uint32_t *cta_v, *cta_t;               // [nctas] totals -> exclusive prefix (in place)
};

__host__ __device__ inline long long align_up(long long x, long long a) {
  return (x + a - 1) / a * a;
}

__host__ McLayout make_layout(int nx, int ny, int nz, void* work) {
  McLayout L;
  L.nx = nx; L.ny = ny; L.nz = nz;
  L.nwz = (nz + 31) / 32;
  L.nwords = (long long)nx * ny * L.nwz;
  L.nctas = (int)((L.nwords + kWordsPerCta - 1) / kWordsPerCta);
  long long wb = align_up(L.nwords * 4, 256);
  char* p = (char*)work;
  L.fx = (uint32_t*)p; p += wb;
  L.fy = (uint32_t*)p; p += wb;
  L.fz = (uint32_t*)p; p += wb;
  L.vpre = (uint32_t*)p; p += wb;
  L.tpre = (uint32_t*)p; p += wb;
  L.sgn = (uint32_t*)p; p += wb;
  long long cb = align_up((long long)L.nctas * 4, 256);
  L.cta_v = (uint32_t*)p; p += cb;
  L.cta_t = (uint32_t*)p; p += cb;
  return L;
}

__device__ __forceinline__ int tri_count(uint64_t packed) {
  // number of 0xF nibbles at the top = clz(~packed)/4 (valid nibbles are <= 11).
  uint64_t inv = ~packed;
  int nf = inv ? (__clzll((long long)inv) >> 2) : 16;
  return (16 - nf) / 3;
}

// Raw loads for the voxels (i,j,32*kw+lane): the four z-rows r0=(i,j) r1=(i+1,j) r2=(i+1,j+1)
// r3=(i,j+1) at k, plus (lane 31 only) at k+1.  Indices are clamped so every lane loads something
// and can take part in the shuffles of cube_index().  Split from the index computation so the
// classify loop can issue the loads of word n+1 before it ballots word n (memory-level
// parallelism: the first version had ~4 loads in flight per warp and ran at 5 % of HBM).
struct CubeLoads {
  float a[4];
  float b[4];  // valid in lane 31 only
};
__device__ __forceinline__ CubeLoads cube_loads(const float* __restrict__ sdf, int nx, int ny,
                                                int nz, int i, int j, int k) {
  const int i1 = min(i + 1, nx - 1), j1 = min(j + 1, ny - 1);
  const int ic = min(i, nx - 1);
  const int kc = min(k, nz - 1);
  const long long snz = nz;
  const float* r0 = sdf + ((long long)ic * ny + j) * snz;
  const float* r1 = sdf + ((long long)i1 * ny + j) * snz;
  const float* r2 = sdf + ((long long)i1 * ny + j1) * snz;
  const float* r3 = sdf + ((long long)ic * ny + j1) * snz;
  CubeLoads c;
  c.a[0] = __ldg(r0 + kc); c.a[1] = __ldg(r1 + kc); c.a[2] = __ldg(r2 + kc); c.a[3] = __ldg(r3 + kc);
  c.b[0] = c.b[1] = c.b[2] = c.b[3] = 0.f;
  if ((threadIdx.x & 31) == 31) {
    const int k1 = min(k + 1, nz - 1);
    c.b[0] = __ldg(r0 + k1); c.b[1] = __ldg(r1 + k1); c.b[2] = __ldg(r2 + k1); c.b[3] = __ldg(r3 + k1);
  }
  return c;
}

// Corner numbering, (x,y,z)=(i,j,k) offsets: c0 000, c1 100, c2 110, c3 010, c4 001, c5 101,
// c6 111, c7 011.  Returns the cube index, or -1 for lanes that are not valid cells.
__device__ __forceinline__ int cube_index(const CubeLoads& c, int nx, int ny, int nz, int i, int j,
                                          int k, float iso, float v[8]) {
  const bool cell = (i < nx - 1) && (j < ny - 1) && (k < nz - 1);
  const bool last = (threadIdx.x & 31) == 31;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const float up = __shfl_down_sync(0xffffffffu, c.a[r], 1);  // value at k+1 from the neighbour lane
    v[r] = c.a[r];
    v[4 + r] = last ? c.b[r] : up;
  }
  if (!cell) return -1;
  int idx = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) idx |= (v[q] < iso) ? (1 << q) : 0;
  return idx;
}

__device__ __forceinline__ int load_cube(const float* __restrict__ sdf, int nx, int ny, int nz,
                                         int i, int j, int k, float iso, float v[8]) {
  const CubeLoads c = cube_loads(sdf, nx, ny, nz, i, j, k);
  return cube_index(c, nx, ny, nz, i, j, k, iso, v);
}

// ---- classification in two passes -------------------------------------------------------------
// Pass 1 (HBM bound, the only full read of the grid): one warp per 32 samples of a z-row, one
// coalesced 128-byte load, `v < iso` balloted into a sign bit-plane (1 bit per sample).
// Pass 2 (one THREAD per 32-cell word): the eight corner bit-words of the word's cells are the sign
// words of rows (i,j) (i+1,j) (i+1,j+1) (i,j+1) and the same shifted by one k; crossed-edge flags are
// XORs of whole words, active cells are where the eight words disagree, and only those cells (a few
// per cent) index the triangle table instead of building a cube index per lane from eight float loads
// (an issue-bound loop).
constexpr int kSignWordsPerWarp = 8;
__global__ void __launch_bounds__(kThreads)
mc_sign_kernel(const float* __restrict__ sdf, McLayout L, float iso) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const long long w0 = warp * kSignWordsPerWarp;
  if (w0 >= L.nwords) return;
  uint32_t row = (uint32_t)(w0 / (uint32_t)L.nwz);
  int kw = (int)(w0 - (long long)row * L.nwz);
  float v[kSignWordsPerWarp];
  bool in[kSignWordsPerWarp];
  uint32_t r = row;
  int q = kw;
#pragma unroll
  for (int u = 0; u < kSignWordsPerWarp; ++u) {   // all loads first: 8 independent 128-byte rows in flight
    const int k = q * 32 + lane;
    in[u] = (w0 + u < L.nwords) && k < L.nz;
    v[u] = in[u] ? __ldg(sdf + (size_t)r * L.nz + k) : 0.f;
    if (++q == L.nwz) { q = 0; ++r; }
  }
#pragma unroll
  for (int u = 0; u < kSignWordsPerWarp; ++u) {
    const uint32_t bits = __ballot_sync(0xffffffffu, in[u] && v[u] < iso);
    if (lane == 0 && w0 + u < L.nwords) L.sgn[w0 + u] = bits;
  }
}

__global__ void __launch_bounds__(kThreads)
mc_classify_kernel(McLayout L) {
  __shared__ uint64_t s_tri[256];
  __shared__ uint32_t s_wv[kWarps], s_wt[kWarps];
  s_tri[threadIdx.x] = kTriPacked[threadIdx.x];   // kThreads == 256
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long word = (long long)blockIdx.x * kWordsPerCta + threadIdx.x;
  uint32_t fx = 0, fy = 0, fz = 0, nv = 0, nt = 0;
  if (word < L.nwords) {
    const uint32_t row = (uint32_t)(word / (uint32_t)L.nwz);
    const int kw = (int)(word - (long long)row * L.nwz);
    const int j = (int)(row % (uint32_t)L.ny), i = (int)(row / (uint32_t)L.ny);
    if (i < L.nx - 1 && j < L.ny - 1) {
      // cells of this word: k = 32 kw + b, valid while k < nz - 1
      const int rem = L.nz - 1 - kw * 32;
      const uint32_t cellmask = rem >= 32 ? 0xffffffffu : (rem > 0 ? ((1u << rem) - 1u) : 0u);
      const bool more = kw + 1 < L.nwz;
      const uint32_t* p0 = L.sgn + word;                       // row (i, j)
      const uint32_t* p1 = p0 + (size_t)L.ny * L.nwz;          // row (i+1, j)
      const uint32_t* p2 = p1 + L.nwz;                         // row (i+1, j+1)
      const uint32_t* p3 = p0 + L.nwz;                         // row (i, j+1)
      const uint32_t a0 = p0[0], a1 = p1[0], a2 = p2[0], a3 = p3[0];
      const uint32_t n0 = more ? p0[1] : 0u, n1 = more ? p1[1] : 0u, n2 = more ? p2[1] : 0u,
                     n3 = more ? p3[1] : 0u;
      // corner bit-words: c0 000, c1 100, c2 110, c3 010 at k; c4..c7 the same rows at k+1
      const uint32_t c[8] = {a0, a1, a2, a3, (a0 >> 1) | (n0 << 31), (a1 >> 1) | (n1 << 31),
                             (a2 >> 1) | (n2 << 31), (a3 >> 1) | (n3 << 31)};
      const uint32_t all_or = c[0] | c[1] | c[2] | c[3] | c[4] | c[5] | c[6] | c[7];
      const uint32_t all_and = c[0] & c[1] & c[2] & c[3] & c[4] & c[5] & c[6] & c[7];
      uint32_t active = cellmask & all_or & ~all_and;
      fx = (c[0] ^ c[1]) & cellmask;   // edge c0-c1 (+x)
      fy = (c[0] ^ c[3]) & cellmask;   // edge c3-c0 (+y)
      fz = (c[0] ^ c[4]) & cellmask;   // edge c0-c4 (+z)
      nv = __popc(fx) + __popc(fy) + __popc(fz);
      while (active) {
        const int b = __ffs(active) - 1;
        active &= active - 1;
        int idx = 0;
#pragma unroll
        for (int qq = 0; qq < 8; ++qq) idx |= ((c[qq] >> b) & 1u) << qq;
        nt += tri_count(s_tri[idx]);
      }
      L.fx[word] = fx; L.fy[word] = fy; L.fz[word] = fz;
    } else {
      L.fx[word] = 0; L.fy[word] = 0; L.fz[word] = 0;
    }
  }
  // CTA-exclusive prefixes of the vertex / triangle counts over the 256 words of this CTA
  uint32_t sv = nv, st = nt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t a = __shfl_up_sync(0xffffffffu, sv, o);
    uint32_t b = __shfl_up_sync(0xffffffffu, st, o);
    if (lane >= o) { sv += a; st += b; }
  }
  if (lane == 31) { s_wv[warp] = sv; s_wt[warp] = st; }
  __syncthreads();
  uint32_t bv = 0, bt = 0;
  for (int w = 0; w < warp; ++w) { bv += s_wv[w]; bt += s_wt[w]; }
  if (word < L.nwords) {
    L.vpre[word] = bv + sv - nv;
    L.tpre[word] = (bt + st - nt) | (nt ? kHasTris : 0u);
  }
  if (threadIdx.x == kThreads - 1) {
    L.cta_v[blockIdx.x] = bv + sv;
    L.cta_t[blockIdx.x] = bt + st;
  }
}

// Single CTA: exclusive scan of the per-CTA totals; grand totals to counts[0..1].
__global__ void __launch_bounds__(1024)
mc_scan_kernel(McLayout L, int32_t* __restrict__ counts) {
  __shared__ uint32_t s_v[32], s_t[32];
  __shared__ uint32_t carry_v, carry_t;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { carry_v = 0; carry_t = 0; }
  __syncthreads();
  for (int base = 0; base < L.nctas; base += 1024) {
    const int i = base + threadIdx.x;
    uint32_t v = i < L.nctas ? L.cta_v[i] : 0u, t = i < L.nctas ? L.cta_t[i] : 0u;
    uint32_t sv = v, st = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t a = __shfl_up_sync(0xffffffffu, sv, o);
      uint32_t b = __shfl_up_sync(0xffffffffu, st, o);
      if (lane >= o) { sv += a; st += b; }
    }
    if (lane == 31) { s_v[warp] = sv; s_t[warp] = st; }
    __syncthreads();
    if (warp == 0) {
      uint32_t a = s_v[lane], b = s_t[lane];
      uint32_t sa = a, sb = b;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        uint32_t x = __shfl_up_sync(0xffffffffu, sa, o);
        uint32_t y = __shfl_up_sync(0xffffffffu, sb, o);
        if (lane >= o) { sa += x; sb += y; }
      }
      s_v[lane] = sa - a; s_t[lane] = sb - b;  // exclusive over warps
    }
    __syncthreads();
    const uint32_t ev = carry_v + s_v[warp] + sv - v;
    const uint32_t et = carry_t + s_t[warp] + st - t;
    if (i < L.nctas) { L.cta_v[i] = ev; L.cta_t[i] = et; }
    __syncthreads();
    if (threadIdx.x == 1023) { carry_v = ev + v; carry_t = et + t; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { counts[0] = (int32_t)carry_v; counts[1] = (int32_t)carry_t; }
}

__device__ __forceinline__ float edge_offset(float v1, float v2, float iso) {
  // reference: double fDelta = v2 - v1 (float subtraction, then widened);
  //            return (iso - v1) / fDelta  (float numerator widened, double division).
  const float fd = __fsub_rn(v2, v1);
  const double delta = (double)fd;
  if (delta == 0.0) return 0.5f;
  return (float)((double)__fsub_rn(iso, v1) / delta);
}

// vertex id of the edge (dir) owned by voxel (oi,oj,ok), -1 when that voxel is not a cell:
//   id = cta_v[word / 256] + vpre[word] + popc(fx, fy, fz below bit k) (+ fx, fy of bit k for dir y, z),
// evaluated from the word records staged in shared memory by mc_emit_kernel: rec[(dx + 2 dy) * 2 + wsel]
// = {fx, fy, fz, cta_v + vpre} of word (i + dx, j + dy, kw + wsel).
__device__ __forceinline__ long long vertex_id_rec(const McLayout& L, const uint4* rec, int kw, int oi, int oj,
                                                   int ok, int row, int dir) {
  if (oi >= L.nx - 1 || oj >= L.ny - 1 || ok >= L.nz - 1) return -1;
  const uint4 r = rec[row * 2 + ((ok >> 5) - kw)];
  const int bit = ok & 31;
  const uint32_t lt = (1u << bit) - 1u;
  uint32_t id = r.w + __popc(r.x & lt) + __popc(r.y & lt) + __popc(r.z & lt);
  if (dir >= 1) id += (r.x >> bit) & 1u;
  if (dir == 2) id += (r.y >> bit) & 1u;
  return (long long)id;
}

__global__ void __launch_bounds__(kThreads)
mc_emit_kernel(const float* __restrict__ sdf, McLayout L, float iso, float xs, float ys, float zs,
               float x0, float y0, float z0, int i_offset, float* __restrict__ verts,
               long long vcap, long long* __restrict__ faces, long long fcap) {
  __shared__ uint4 s_rec[kWarps][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long word0 = (long long)blockIdx.x * kWordsPerCta + (long long)warp * kWordsPerWarp;
  const uint32_t cta_v = L.cta_v[blockIdx.x], cta_t = L.cta_t[blockIdx.x];
  // one coalesced read of this warp's 32 word records
  uint32_t wfx = 0, wfy = 0, wfz = 0, wv = 0, wt = 0;
  {
    const long long w = word0 + lane;
    if (w < L.nwords) {
      wfx = L.fx[w]; wfy = L.fy[w]; wfz = L.fz[w]; wv = L.vpre[w]; wt = L.tpre[w];
    }
  }
  // words that own a vertex or hold faces (a word can hold faces but own no vertex: all its crossed
  // edges belong to neighbours, hence the separate has-triangles bit); the rest cost nothing
  uint32_t todo = __ballot_sync(0xffffffffu, (wfx | wfy | wfz) != 0u || (wt & kHasTris) != 0u);
  while (todo) {
    const int it = __ffs(todo) - 1;
    todo &= todo - 1;
    const long long word = word0 + it;
    const uint32_t fx = __shfl_sync(0xffffffffu, wfx, it), fy = __shfl_sync(0xffffffffu, wfy, it),
                   fz = __shfl_sync(0xffffffffu, wfz, it);
    const uint32_t tp = __shfl_sync(0xffffffffu, wt, it);
    const uint32_t vbase = cta_v + __shfl_sync(0xffffffffu, wv, it);
    const uint32_t tbase = cta_t + (tp & ~kHasTris);
    const int kw = (int)((uint32_t)word % (uint32_t)L.nwz);
    const uint32_t ij = (uint32_t)word / (uint32_t)L.nwz;
    const int j = (int)(ij % (uint32_t)L.ny), i = (int)(ij / (uint32_t)L.ny);
    const int k = kw * 32 + lane;
    float v[8];
    const int idx = load_cube(sdf, L.nx, L.ny, L.nz, i, j, k, iso, v);
    // records of the eight words the faces of this word can reference: rows (i,j) (i+1,j) (i,j+1)
    // (i+1,j+1) at kw and kw+1, fetched once by lanes 0..7 instead of five loads per face corner
    __syncwarp();
    if (lane < 8) {
      const int row = lane >> 1, ws = lane & 1;
      const int oi = i + (row & 1), oj = j + (row >> 1);
      uint4 r = make_uint4(0u, 0u, 0u, 0u);
      if (oi < L.nx && oj < L.ny && kw + ws < L.nwz) {
        const uint32_t w = ((uint32_t)oi * (uint32_t)L.ny + (uint32_t)oj) * (uint32_t)L.nwz + (uint32_t)(kw + ws);
        r = make_uint4(__ldg(L.fx + w), __ldg(L.fy + w), __ldg(L.fz + w),
                       __ldg(L.cta_v + (w / kWordsPerCta)) + __ldg(L.vpre + w));
      }
      s_rec[warp][lane] = r;
    }
    __syncwarp();
    // ---- vertices owned by this voxel, ordered (k, dir)
    const uint32_t bitm = 1u << lane, lt = bitm - 1u;
    if ((fx | fy | fz) & bitm) {
      long long vid = (long long)vbase + __popc(fx & lt) + __popc(fy & lt) + __popc(fz & lt);
      const float fi = (float)(i + i_offset), fj = (float)j, fk = (float)k;
      if (fx & bitm) {
        const float t = edge_offset(v[0], v[1], iso);
        if (vid < vcap) {
          verts[vid * 3 + 0] = fmaf(__fadd_rn(fi, __fadd_rn(0.0f, t)), xs, x0);
          verts[vid * 3 + 1] = fmaf(fj, ys, y0);
          verts[vid * 3 + 2] = fmaf(fk, zs, z0);
        }
        ++vid;
      }
      if (fy & bitm) {
        const float t = edge_offset(v[3], v[0], iso);  // edge 3: corner 3 -> corner 0
        if (vid < vcap) {
          verts[vid * 3 + 0] = fmaf(fi, xs, x0);
          verts[vid * 3 + 1] = fmaf(__fadd_rn(fj, __fsub_rn(1.0f, t)), ys, y0);
          verts[vid * 3 + 2] = fmaf(fk, zs, z0);
        }
        ++vid;
      }
      if (fz & bitm) {
        const float t = edge_offset(v[0], v[4], iso);
        if (vid < vcap) {
          verts[vid * 3 + 0] = fmaf(fi, xs, x0);
          verts[vid * 3 + 1] = fmaf(fj, ys, y0);
          verts[vid * 3 + 2] = fmaf(__fadd_rn(fk, __fadd_rn(0.0f, t)), zs, z0);
        }
      }
    }
    // ---- faces of this voxel, ordered (k, triangle#)
    const bool has = idx > 0 && idx < 255;
    const uint64_t packed = has ? kTriPacked[idx] : ~0ull;
    const int nt = has ? tri_count(packed) : 0;
    int sc = nt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int a = __shfl_up_sync(0xffffffffu, sc, o);
      if (lane >= o) sc += a;
    }
    long long fid = (long long)tbase + (sc - nt);
    for (int t = 0; t < nt; ++t, ++fid) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int e = (int)((packed >> (4 * (3 * t + c))) & 0xF);
        // edge -> owner voxel offset and direction:
        //   +x for edges 1,5,9,10 ; +y for 2,6,10,11 ; +z for 4,5,6,7
        //   dir = z for e>=8, else y for odd e, x for even e.
        const int dx = (0x622 >> e) & 1;
        const int dy = (0xC44 >> e) & 1;
        const int dz = (0x0F0 >> e) & 1;
        const int dir = e >= 8 ? 2 : (e & 1);
        const long long id = vertex_id_rec(L, s_rec[warp], kw, i + dx, j + dy, k + dz, dx + 2 * dy, dir);
        if (fid < fcap) faces[fid * 3 + (2 - c)] = id;
      }
    }
  }
}

}  // namespace

extern "C" {

int64_t sr_mc_work_bytes(int nx, int ny, int nz) {
  if (nx <= 0 || ny <= 0 || nz <= 0) return 0;
  long long nwz = (nz + 31) / 32;
  long long nwords = (long long)nx * ny * nwz;
  long long nctas = (nwords + kWordsPerCta - 1) / kWordsPerCta;
  return 6 * align_up(nwords * 4, 256) + 2 * align_up(nctas * 4, 256);
}

int sr_mc_count(const float* sdf, int nx, int ny, int nz, float iso, void* work, int32_t* counts,
                cudaStream_t s) {
  if (nx <= 0 || ny <= 0 || nz <= 0 || !sdf || !work || !counts) return SR_EINVAL;
  if ((long long)nx * ny * nz > 0x7fffffffLL) return SR_EUNSUPPORTED;
  McLayout L = make_layout(nx, ny, nz, work);
  {
    const long long warps = (L.nwords + kSignWordsPerWarp - 1) / kSignWordsPerWarp;
    mc_sign_kernel<<<(unsigned)((warps + kWarps - 1) / kWarps), kThreads, 0, s>>>(sdf, L, iso);
  }
  mc_classify_kernel<<<L.nctas, kThreads, 0, s>>>(L);
  mc_scan_kernel<<<1, 1024, 0, s>>>(L, counts);
  return sr_launch_status();
}

int sr_mc_emit(const float* sdf, int nx, int ny, int nz, float iso, float xstep, float ystep,
               float zstep, float xmin, float ymin, float zmin, int i_offset, const void* work,
               float* vertices, int64_t vcap, int64_t* faces, int64_t fcap, cudaStream_t s) {
  if (nx <= 0 || ny <= 0 || nz <= 0 || !sdf || !work) return SR_EINVAL;
  if ((vcap > 0 && !vertices) || (fcap > 0 && !faces)) return SR_EINVAL;
  if (vcap == 0 && fcap == 0) return SR_OK;
  McLayout L = make_layout(nx, ny, nz, const_cast<void*>(work));
  mc_emit_kernel<<<L.nctas, kThreads, 0, s>>>(sdf, L, iso, xstep, ystep, zstep, xmin, ymin, zmin,
                                               i_offset, vertices, (long long)vcap, (long long*)faces,
                                               (long long)fcap);
  return sr_launch_status();
}
}
