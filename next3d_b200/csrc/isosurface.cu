// Marching cubes on a float32 grid g[a0, a1, a2] of shape [nz, ny, nx] (next3d_b200/isosurface.py; DESIGN.md section 3.7).
// The mesh is a function of the grid and the level alone (tests/isosurface_oracle.py restates it in numpy):
//   iso_count_rows   one warp per voxel row (a0, a1), 32 voxels at a time: the row's crossed edges (one vertex each, owned by the
//                    edge's lower endpoint), the triangles of its cells (c_tri) and its non-finite voxels.
//   iso_scan_tiles   one block per tile of kTile rows: the tile's three sums.
//   iso_scan_rows    one block per tile: the sums of the tiles before it, then the tile's rows scanned in place into exclusive
//                    offsets; the last tile writes the totals {vertices, triangles, non-finite voxels}.
//   iso_emit_rows    one warp per voxel row, 31 voxels at a time (lane 31 reads the next voxel for lane 30): the in-row prefixes
//                    of the (up to four) rows a cell touches, recomputed from the grid, give every vertex id; the row's vertices
//                    and the triangles of its cells go to the row offsets.
// The workspace holds three int64 per row and per tile, never a per-voxel array.
#include "common.cuh"

namespace {

constexpr int kWarps = 8;                 // warps per block of the row kernels
constexpr int kScanThreads = 1024;
constexpr int kTile = 4 * kScanThreads;   // rows per scan tile

// Triangles of the 256 cell configurations (sum of inside(k) << k over corners k = dx + 2 dy + 4 dz): up to five triangles of
// three edge numbers, -1 past the last, and the triangle count in byte 15.  Derived from the face rule of DESIGN.md section 3.7;
// tests/test_isosurface_cpu.py derives it again and compares.
__device__ __align__(16) const int8_t c_tri[256][16] = {
    {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 0},   //   0
    { 0,  4,  8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   //   1
    { 0,  9,  5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   //   2
    { 4,  8,  9,  4,  9,  5, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //   3
    { 1, 10,  4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   //   4
    { 0,  1, 10,  0, 10,  8, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //   5
    { 0,  9,  5,  1, 10,  4, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //   6
    { 1, 10,  8,  1,  8,  9,  1,  9,  5, -1, -1, -1, -1, -1, -1, 3},   //   7
    { 1,  5, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   //   8
    { 0,  4,  8,  1,  5, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //   9
    { 0,  9, 11,  0, 11,  1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  10
    { 1,  4,  8,  1,  8,  9,  1,  9, 11, -1, -1, -1, -1, -1, -1, 3},   //  11
    { 4,  5, 11,  4, 11, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  12
    { 0,  5, 11,  0, 11, 10,  0, 10,  8, -1, -1, -1, -1, -1, -1, 3},   //  13
    { 0,  9, 11,  0, 11, 10,  0, 10,  4, -1, -1, -1, -1, -1, -1, 3},   //  14
    { 8,  9, 11,  8, 11, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  15
    { 2,  8,  6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   //  16
    { 0,  4,  6,  0,  6,  2, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  17
    { 0,  9,  5,  2,  8,  6, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  18
    { 2,  9,  5,  2,  5,  4,  2,  4,  6, -1, -1, -1, -1, -1, -1, 3},   //  19
    { 1, 10,  4,  2,  8,  6, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  20
    { 0,  1, 10,  0, 10,  6,  0,  6,  2, -1, -1, -1, -1, -1, -1, 3},   //  21
    { 0,  9,  5,  1, 10,  4,  2,  8,  6, -1, -1, -1, -1, -1, -1, 3},   //  22
    { 1, 10,  6,  1,  6,  2,  1,  2,  9,  1,  9,  5, -1, -1, -1, 4},   //  23
    { 1,  5, 11,  2,  8,  6, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  24
    { 0,  4,  6,  0,  6,  2,  1,  5, 11, -1, -1, -1, -1, -1, -1, 3},   //  25
    { 0,  9, 11,  0, 11,  1,  2,  8,  6, -1, -1, -1, -1, -1, -1, 3},   //  26
    { 1,  4,  6,  1,  6,  2,  1,  2,  9,  1,  9, 11, -1, -1, -1, 4},   //  27
    { 2,  8,  6,  4,  5, 11,  4, 11, 10, -1, -1, -1, -1, -1, -1, 3},   //  28
    { 0,  5, 11,  0, 11, 10,  0, 10,  6,  0,  6,  2, -1, -1, -1, 4},   //  29
    { 0,  9, 11,  0, 11, 10,  0, 10,  4,  2,  8,  6, -1, -1, -1, 4},   //  30
    { 2,  9, 11,  2, 11, 10,  2, 10,  6, -1, -1, -1, -1, -1, -1, 3},   //  31
    { 2,  7,  9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   //  32
    { 0,  4,  8,  2,  7,  9, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  33
    { 0,  2,  7,  0,  7,  5, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  34
    { 2,  7,  5,  2,  5,  4,  2,  4,  8, -1, -1, -1, -1, -1, -1, 3},   //  35
    { 1, 10,  4,  2,  7,  9, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  36
    { 0,  1, 10,  0, 10,  8,  2,  7,  9, -1, -1, -1, -1, -1, -1, 3},   //  37
    { 0,  2,  7,  0,  7,  5,  1, 10,  4, -1, -1, -1, -1, -1, -1, 3},   //  38
    { 1, 10,  8,  1,  8,  2,  1,  2,  7,  1,  7,  5, -1, -1, -1, 4},   //  39
    { 1,  5, 11,  2,  7,  9, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  40
    { 0,  4,  8,  1,  5, 11,  2,  7,  9, -1, -1, -1, -1, -1, -1, 3},   //  41
    { 0,  2,  7,  0,  7, 11,  0, 11,  1, -1, -1, -1, -1, -1, -1, 3},   //  42
    { 1,  4,  8,  1,  8,  2,  1,  2,  7,  1,  7, 11, -1, -1, -1, 4},   //  43
    { 2,  7,  9,  4,  5, 11,  4, 11, 10, -1, -1, -1, -1, -1, -1, 3},   //  44
    { 0,  5, 11,  0, 11, 10,  0, 10,  8,  2,  7,  9, -1, -1, -1, 4},   //  45
    { 0,  2,  7,  0,  7, 11,  0, 11, 10,  0, 10,  4, -1, -1, -1, 4},   //  46
    { 2,  7, 11,  2, 11, 10,  2, 10,  8, -1, -1, -1, -1, -1, -1, 3},   //  47
    { 6,  7,  9,  6,  9,  8, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  48
    { 0,  4,  6,  0,  6,  7,  0,  7,  9, -1, -1, -1, -1, -1, -1, 3},   //  49
    { 0,  8,  6,  0,  6,  7,  0,  7,  5, -1, -1, -1, -1, -1, -1, 3},   //  50
    { 4,  6,  7,  4,  7,  5, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  51
    { 1, 10,  4,  6,  7,  9,  6,  9,  8, -1, -1, -1, -1, -1, -1, 3},   //  52
    { 0,  1, 10,  0, 10,  6,  0,  6,  7,  0,  7,  9, -1, -1, -1, 4},   //  53
    { 0,  8,  6,  0,  6,  7,  0,  7,  5,  1, 10,  4, -1, -1, -1, 4},   //  54
    { 1, 10,  6,  1,  6,  7,  1,  7,  5, -1, -1, -1, -1, -1, -1, 3},   //  55
    { 1,  5, 11,  6,  7,  9,  6,  9,  8, -1, -1, -1, -1, -1, -1, 3},   //  56
    { 0,  4,  6,  0,  6,  7,  0,  7,  9,  1,  5, 11, -1, -1, -1, 4},   //  57
    { 0,  8,  6,  0,  6,  7,  0,  7, 11,  0, 11,  1, -1, -1, -1, 4},   //  58
    { 1,  4,  6,  1,  6,  7,  1,  7, 11, -1, -1, -1, -1, -1, -1, 3},   //  59
    { 4,  5, 11,  4, 11, 10,  6,  7,  9,  6,  9,  8, -1, -1, -1, 4},   //  60
    { 0,  5, 11,  0, 11, 10,  0, 10,  6,  0,  6,  7,  0,  7,  9, 5},   //  61
    { 0,  8,  6,  0,  6,  7,  0,  7, 11,  0, 11, 10,  0, 10,  4, 5},   //  62
    { 6,  7, 11,  6, 11, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  63
    { 3,  6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   //  64
    { 0,  4,  8,  3,  6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  65
    { 0,  9,  5,  3,  6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  66
    { 3,  6, 10,  4,  8,  9,  4,  9,  5, -1, -1, -1, -1, -1, -1, 3},   //  67
    { 1,  3,  6,  1,  6,  4, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  68
    { 0,  1,  3,  0,  3,  6,  0,  6,  8, -1, -1, -1, -1, -1, -1, 3},   //  69
    { 0,  9,  5,  1,  3,  6,  1,  6,  4, -1, -1, -1, -1, -1, -1, 3},   //  70
    { 1,  3,  6,  1,  6,  8,  1,  8,  9,  1,  9,  5, -1, -1, -1, 4},   //  71
    { 1,  5, 11,  3,  6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  72
    { 0,  4,  8,  1,  5, 11,  3,  6, 10, -1, -1, -1, -1, -1, -1, 3},   //  73
    { 0,  9, 11,  0, 11,  1,  3,  6, 10, -1, -1, -1, -1, -1, -1, 3},   //  74
    { 1,  4,  8,  1,  8,  9,  1,  9, 11,  3,  6, 10, -1, -1, -1, 4},   //  75
    { 3,  6,  4,  3,  4,  5,  3,  5, 11, -1, -1, -1, -1, -1, -1, 3},   //  76
    { 0,  5, 11,  0, 11,  3,  0,  3,  6,  0,  6,  8, -1, -1, -1, 4},   //  77
    { 0,  9, 11,  0, 11,  3,  0,  3,  6,  0,  6,  4, -1, -1, -1, 4},   //  78
    { 3,  6,  8,  3,  8,  9,  3,  9, 11, -1, -1, -1, -1, -1, -1, 3},   //  79
    { 2,  8, 10,  2, 10,  3, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  80
    { 0,  4, 10,  0, 10,  3,  0,  3,  2, -1, -1, -1, -1, -1, -1, 3},   //  81
    { 0,  9,  5,  2,  8, 10,  2, 10,  3, -1, -1, -1, -1, -1, -1, 3},   //  82
    { 2,  9,  5,  2,  5,  4,  2,  4, 10,  2, 10,  3, -1, -1, -1, 4},   //  83
    { 1,  3,  2,  1,  2,  8,  1,  8,  4, -1, -1, -1, -1, -1, -1, 3},   //  84
    { 0,  1,  3,  0,  3,  2, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  85
    { 0,  9,  5,  1,  3,  2,  1,  2,  8,  1,  8,  4, -1, -1, -1, 4},   //  86
    { 1,  3,  2,  1,  2,  9,  1,  9,  5, -1, -1, -1, -1, -1, -1, 3},   //  87
    { 1,  5, 11,  2,  8, 10,  2, 10,  3, -1, -1, -1, -1, -1, -1, 3},   //  88
    { 0,  4, 10,  0, 10,  3,  0,  3,  2,  1,  5, 11, -1, -1, -1, 4},   //  89
    { 0,  9, 11,  0, 11,  1,  2,  8, 10,  2, 10,  3, -1, -1, -1, 4},   //  90
    { 4, 10,  3,  4,  3,  2,  4,  2,  9,  4,  9, 11,  4, 11,  1, 5},   //  91
    { 2,  8,  4,  2,  4,  5,  2,  5, 11,  2, 11,  3, -1, -1, -1, 4},   //  92
    { 0,  5, 11,  0, 11,  3,  0,  3,  2, -1, -1, -1, -1, -1, -1, 3},   //  93
    {11,  3,  2, 11,  2,  8, 11,  8,  4, 11,  4,  0, 11,  0,  9, 5},   //  94
    { 2,  9, 11,  2, 11,  3, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  95
    { 2,  7,  9,  3,  6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   //  96
    { 0,  4,  8,  2,  7,  9,  3,  6, 10, -1, -1, -1, -1, -1, -1, 3},   //  97
    { 0,  2,  7,  0,  7,  5,  3,  6, 10, -1, -1, -1, -1, -1, -1, 3},   //  98
    { 2,  7,  5,  2,  5,  4,  2,  4,  8,  3,  6, 10, -1, -1, -1, 4},   //  99
    { 1,  3,  6,  1,  6,  4,  2,  7,  9, -1, -1, -1, -1, -1, -1, 3},   // 100
    { 0,  1,  3,  0,  3,  6,  0,  6,  8,  2,  7,  9, -1, -1, -1, 4},   // 101
    { 0,  2,  7,  0,  7,  5,  1,  3,  6,  1,  6,  4, -1, -1, -1, 4},   // 102
    { 1,  3,  6,  1,  6,  8,  1,  8,  2,  1,  2,  7,  1,  7,  5, 5},   // 103
    { 1,  5, 11,  2,  7,  9,  3,  6, 10, -1, -1, -1, -1, -1, -1, 3},   // 104
    { 0,  4,  8,  1,  5, 11,  2,  7,  9,  3,  6, 10, -1, -1, -1, 4},   // 105
    { 0,  2,  7,  0,  7, 11,  0, 11,  1,  3,  6, 10, -1, -1, -1, 4},   // 106
    { 1,  4,  8,  1,  8,  2,  1,  2,  7,  1,  7, 11,  3,  6, 10, 5},   // 107
    { 2,  7,  9,  3,  6,  4,  3,  4,  5,  3,  5, 11, -1, -1, -1, 4},   // 108
    { 0,  5, 11,  0, 11,  3,  0,  3,  6,  0,  6,  8,  2,  7,  9, 5},   // 109
    { 0,  2,  7,  0,  7, 11,  0, 11,  3,  0,  3,  6,  0,  6,  4, 5},   // 110
    {11,  3,  6, 11,  6,  8, 11,  8,  2, 11,  2,  7, -1, -1, -1, 4},   // 111
    { 3,  7,  9,  3,  9,  8,  3,  8, 10, -1, -1, -1, -1, -1, -1, 3},   // 112
    { 0,  4, 10,  0, 10,  3,  0,  3,  7,  0,  7,  9, -1, -1, -1, 4},   // 113
    { 0,  8, 10,  0, 10,  3,  0,  3,  7,  0,  7,  5, -1, -1, -1, 4},   // 114
    { 3,  7,  5,  3,  5,  4,  3,  4, 10, -1, -1, -1, -1, -1, -1, 3},   // 115
    { 1,  3,  7,  1,  7,  9,  1,  9,  8,  1,  8,  4, -1, -1, -1, 4},   // 116
    { 0,  1,  3,  0,  3,  7,  0,  7,  9, -1, -1, -1, -1, -1, -1, 3},   // 117
    { 8,  4,  1,  8,  1,  3,  8,  3,  7,  8,  7,  5,  8,  5,  0, 5},   // 118
    { 1,  3,  7,  1,  7,  5, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 119
    { 1,  5, 11,  3,  7,  9,  3,  9,  8,  3,  8, 10, -1, -1, -1, 4},   // 120
    { 0,  4, 10,  0, 10,  3,  0,  3,  7,  0,  7,  9,  1,  5, 11, 5},   // 121
    { 0,  8, 10,  0, 10,  3,  0,  3,  7,  0,  7, 11,  0, 11,  1, 5},   // 122
    { 4, 10,  3,  4,  3,  7,  4,  7, 11,  4, 11,  1, -1, -1, -1, 4},   // 123
    { 3,  7,  9,  3,  9,  8,  3,  8,  4,  3,  4,  5,  3,  5, 11, 5},   // 124
    { 0,  5, 11,  0, 11,  3,  0,  3,  7,  0,  7,  9, -1, -1, -1, 4},   // 125
    { 0,  8,  4,  3,  7, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 126
    { 3,  7, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   // 127
    { 3, 11,  7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   // 128
    { 0,  4,  8,  3, 11,  7, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 129
    { 0,  9,  5,  3, 11,  7, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 130
    { 3, 11,  7,  4,  8,  9,  4,  9,  5, -1, -1, -1, -1, -1, -1, 3},   // 131
    { 1, 10,  4,  3, 11,  7, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 132
    { 0,  1, 10,  0, 10,  8,  3, 11,  7, -1, -1, -1, -1, -1, -1, 3},   // 133
    { 0,  9,  5,  1, 10,  4,  3, 11,  7, -1, -1, -1, -1, -1, -1, 3},   // 134
    { 1, 10,  8,  1,  8,  9,  1,  9,  5,  3, 11,  7, -1, -1, -1, 4},   // 135
    { 1,  5,  7,  1,  7,  3, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 136
    { 0,  4,  8,  1,  5,  7,  1,  7,  3, -1, -1, -1, -1, -1, -1, 3},   // 137
    { 0,  9,  7,  0,  7,  3,  0,  3,  1, -1, -1, -1, -1, -1, -1, 3},   // 138
    { 1,  4,  8,  1,  8,  9,  1,  9,  7,  1,  7,  3, -1, -1, -1, 4},   // 139
    { 3, 10,  4,  3,  4,  5,  3,  5,  7, -1, -1, -1, -1, -1, -1, 3},   // 140
    { 0,  5,  7,  0,  7,  3,  0,  3, 10,  0, 10,  8, -1, -1, -1, 4},   // 141
    { 0,  9,  7,  0,  7,  3,  0,  3, 10,  0, 10,  4, -1, -1, -1, 4},   // 142
    { 3, 10,  8,  3,  8,  9,  3,  9,  7, -1, -1, -1, -1, -1, -1, 3},   // 143
    { 2,  8,  6,  3, 11,  7, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 144
    { 0,  4,  6,  0,  6,  2,  3, 11,  7, -1, -1, -1, -1, -1, -1, 3},   // 145
    { 0,  9,  5,  2,  8,  6,  3, 11,  7, -1, -1, -1, -1, -1, -1, 3},   // 146
    { 2,  9,  5,  2,  5,  4,  2,  4,  6,  3, 11,  7, -1, -1, -1, 4},   // 147
    { 1, 10,  4,  2,  8,  6,  3, 11,  7, -1, -1, -1, -1, -1, -1, 3},   // 148
    { 0,  1, 10,  0, 10,  6,  0,  6,  2,  3, 11,  7, -1, -1, -1, 4},   // 149
    { 0,  9,  5,  1, 10,  4,  2,  8,  6,  3, 11,  7, -1, -1, -1, 4},   // 150
    { 1, 10,  6,  1,  6,  2,  1,  2,  9,  1,  9,  5,  3, 11,  7, 5},   // 151
    { 1,  5,  7,  1,  7,  3,  2,  8,  6, -1, -1, -1, -1, -1, -1, 3},   // 152
    { 0,  4,  6,  0,  6,  2,  1,  5,  7,  1,  7,  3, -1, -1, -1, 4},   // 153
    { 0,  9,  7,  0,  7,  3,  0,  3,  1,  2,  8,  6, -1, -1, -1, 4},   // 154
    { 1,  4,  6,  1,  6,  2,  1,  2,  9,  1,  9,  7,  1,  7,  3, 5},   // 155
    { 2,  8,  6,  3, 10,  4,  3,  4,  5,  3,  5,  7, -1, -1, -1, 4},   // 156
    { 0,  5,  7,  0,  7,  3,  0,  3, 10,  0, 10,  6,  0,  6,  2, 5},   // 157
    { 0,  9,  7,  0,  7,  3,  0,  3, 10,  0, 10,  4,  2,  8,  6, 5},   // 158
    { 9,  7,  3,  9,  3, 10,  9, 10,  6,  9,  6,  2, -1, -1, -1, 4},   // 159
    { 2,  3, 11,  2, 11,  9, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 160
    { 0,  4,  8,  2,  3, 11,  2, 11,  9, -1, -1, -1, -1, -1, -1, 3},   // 161
    { 0,  2,  3,  0,  3, 11,  0, 11,  5, -1, -1, -1, -1, -1, -1, 3},   // 162
    { 2,  3, 11,  2, 11,  5,  2,  5,  4,  2,  4,  8, -1, -1, -1, 4},   // 163
    { 1, 10,  4,  2,  3, 11,  2, 11,  9, -1, -1, -1, -1, -1, -1, 3},   // 164
    { 0,  1, 10,  0, 10,  8,  2,  3, 11,  2, 11,  9, -1, -1, -1, 4},   // 165
    { 0,  2,  3,  0,  3, 11,  0, 11,  5,  1, 10,  4, -1, -1, -1, 4},   // 166
    { 8,  2,  3,  8,  3, 11,  8, 11,  5,  8,  5,  1,  8,  1, 10, 5},   // 167
    { 1,  5,  9,  1,  9,  2,  1,  2,  3, -1, -1, -1, -1, -1, -1, 3},   // 168
    { 0,  4,  8,  1,  5,  9,  1,  9,  2,  1,  2,  3, -1, -1, -1, 4},   // 169
    { 0,  2,  3,  0,  3,  1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 170
    { 1,  4,  8,  1,  8,  2,  1,  2,  3, -1, -1, -1, -1, -1, -1, 3},   // 171
    { 2,  3, 10,  2, 10,  4,  2,  4,  5,  2,  5,  9, -1, -1, -1, 4},   // 172
    { 5,  9,  2,  5,  2,  3,  5,  3, 10,  5, 10,  8,  5,  8,  0, 5},   // 173
    { 0,  2,  3,  0,  3, 10,  0, 10,  4, -1, -1, -1, -1, -1, -1, 3},   // 174
    { 2,  3, 10,  2, 10,  8, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 175
    { 3, 11,  9,  3,  9,  8,  3,  8,  6, -1, -1, -1, -1, -1, -1, 3},   // 176
    { 0,  4,  6,  0,  6,  3,  0,  3, 11,  0, 11,  9, -1, -1, -1, 4},   // 177
    { 0,  8,  6,  0,  6,  3,  0,  3, 11,  0, 11,  5, -1, -1, -1, 4},   // 178
    { 3, 11,  5,  3,  5,  4,  3,  4,  6, -1, -1, -1, -1, -1, -1, 3},   // 179
    { 1, 10,  4,  3, 11,  9,  3,  9,  8,  3,  8,  6, -1, -1, -1, 4},   // 180
    { 0,  1, 10,  0, 10,  6,  0,  6,  3,  0,  3, 11,  0, 11,  9, 5},   // 181
    { 0,  8,  6,  0,  6,  3,  0,  3, 11,  0, 11,  5,  1, 10,  4, 5},   // 182
    { 6,  3, 11,  6, 11,  5,  6,  5,  1,  6,  1, 10, -1, -1, -1, 4},   // 183
    { 1,  5,  9,  1,  9,  8,  1,  8,  6,  1,  6,  3, -1, -1, -1, 4},   // 184
    { 6,  3,  1,  6,  1,  5,  6,  5,  9,  6,  9,  0,  6,  0,  4, 5},   // 185
    { 0,  8,  6,  0,  6,  3,  0,  3,  1, -1, -1, -1, -1, -1, -1, 3},   // 186
    { 1,  4,  6,  1,  6,  3, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 187
    { 3, 10,  4,  3,  4,  5,  3,  5,  9,  3,  9,  8,  3,  8,  6, 5},   // 188
    { 0,  5,  9,  3, 10,  6, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 189
    { 0,  8,  6,  0,  6,  3,  0,  3, 10,  0, 10,  4, -1, -1, -1, 4},   // 190
    { 3, 10,  6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   // 191
    { 6, 10, 11,  6, 11,  7, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 192
    { 0,  4,  8,  6, 10, 11,  6, 11,  7, -1, -1, -1, -1, -1, -1, 3},   // 193
    { 0,  9,  5,  6, 10, 11,  6, 11,  7, -1, -1, -1, -1, -1, -1, 3},   // 194
    { 4,  8,  9,  4,  9,  5,  6, 10, 11,  6, 11,  7, -1, -1, -1, 4},   // 195
    { 1, 11,  7,  1,  7,  6,  1,  6,  4, -1, -1, -1, -1, -1, -1, 3},   // 196
    { 0,  1, 11,  0, 11,  7,  0,  7,  6,  0,  6,  8, -1, -1, -1, 4},   // 197
    { 0,  9,  5,  1, 11,  7,  1,  7,  6,  1,  6,  4, -1, -1, -1, 4},   // 198
    { 1, 11,  7,  1,  7,  6,  1,  6,  8,  1,  8,  9,  1,  9,  5, 5},   // 199
    { 1,  5,  7,  1,  7,  6,  1,  6, 10, -1, -1, -1, -1, -1, -1, 3},   // 200
    { 0,  4,  8,  1,  5,  7,  1,  7,  6,  1,  6, 10, -1, -1, -1, 4},   // 201
    { 0,  9,  7,  0,  7,  6,  0,  6, 10,  0, 10,  1, -1, -1, -1, 4},   // 202
    { 1,  4,  8,  1,  8,  9,  1,  9,  7,  1,  7,  6,  1,  6, 10, 5},   // 203
    { 4,  5,  7,  4,  7,  6, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 204
    { 0,  5,  7,  0,  7,  6,  0,  6,  8, -1, -1, -1, -1, -1, -1, 3},   // 205
    { 0,  9,  7,  0,  7,  6,  0,  6,  4, -1, -1, -1, -1, -1, -1, 3},   // 206
    { 6,  8,  9,  6,  9,  7, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 207
    { 2,  8, 10,  2, 10, 11,  2, 11,  7, -1, -1, -1, -1, -1, -1, 3},   // 208
    { 0,  4, 10,  0, 10, 11,  0, 11,  7,  0,  7,  2, -1, -1, -1, 4},   // 209
    { 0,  9,  5,  2,  8, 10,  2, 10, 11,  2, 11,  7, -1, -1, -1, 4},   // 210
    { 2,  9,  5,  2,  5,  4,  2,  4, 10,  2, 10, 11,  2, 11,  7, 5},   // 211
    { 1, 11,  7,  1,  7,  2,  1,  2,  8,  1,  8,  4, -1, -1, -1, 4},   // 212
    { 0,  1, 11,  0, 11,  7,  0,  7,  2, -1, -1, -1, -1, -1, -1, 3},   // 213
    { 0,  9,  5,  1, 11,  7,  1,  7,  2,  1,  2,  8,  1,  8,  4, 5},   // 214
    { 1, 11,  7,  1,  7,  2,  1,  2,  9,  1,  9,  5, -1, -1, -1, 4},   // 215
    { 1,  5,  7,  1,  7,  2,  1,  2,  8,  1,  8, 10, -1, -1, -1, 4},   // 216
    {10,  1,  5, 10,  5,  7, 10,  7,  2, 10,  2,  0, 10,  0,  4, 5},   // 217
    { 7,  2,  8,  7,  8, 10,  7, 10,  1,  7,  1,  0,  7,  0,  9, 5},   // 218
    { 1,  4, 10,  2,  9,  7, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 219
    { 2,  8,  4,  2,  4,  5,  2,  5,  7, -1, -1, -1, -1, -1, -1, 3},   // 220
    { 0,  5,  7,  0,  7,  2, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 221
    { 7,  2,  8,  7,  8,  4,  7,  4,  0,  7,  0,  9, -1, -1, -1, 4},   // 222
    { 2,  9,  7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   // 223
    { 2,  6, 10,  2, 10, 11,  2, 11,  9, -1, -1, -1, -1, -1, -1, 3},   // 224
    { 0,  4,  8,  2,  6, 10,  2, 10, 11,  2, 11,  9, -1, -1, -1, 4},   // 225
    { 0,  2,  6,  0,  6, 10,  0, 10, 11,  0, 11,  5, -1, -1, -1, 4},   // 226
    { 2,  6, 10,  2, 10, 11,  2, 11,  5,  2,  5,  4,  2,  4,  8, 5},   // 227
    { 1, 11,  9,  1,  9,  2,  1,  2,  6,  1,  6,  4, -1, -1, -1, 4},   // 228
    { 1, 11,  9,  1,  9,  2,  1,  2,  6,  1,  6,  8,  1,  8,  0, 5},   // 229
    { 2,  6,  4,  2,  4,  1,  2,  1, 11,  2, 11,  5,  2,  5,  0, 5},   // 230
    { 1, 11,  5,  2,  6,  8, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 231
    { 1,  5,  9,  1,  9,  2,  1,  2,  6,  1,  6, 10, -1, -1, -1, 4},   // 232
    { 0,  4,  8,  1,  5,  9,  1,  9,  2,  1,  2,  6,  1,  6, 10, 5},   // 233
    { 0,  2,  6,  0,  6, 10,  0, 10,  1, -1, -1, -1, -1, -1, -1, 3},   // 234
    { 1,  4,  8,  1,  8,  2,  1,  2,  6,  1,  6, 10, -1, -1, -1, 4},   // 235
    { 2,  6,  4,  2,  4,  5,  2,  5,  9, -1, -1, -1, -1, -1, -1, 3},   // 236
    { 5,  9,  2,  5,  2,  6,  5,  6,  8,  5,  8,  0, -1, -1, -1, 4},   // 237
    { 0,  2,  6,  0,  6,  4, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 238
    { 2,  6,  8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   // 239
    { 8, 10, 11,  8, 11,  9, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 240
    { 0,  4, 10,  0, 10, 11,  0, 11,  9, -1, -1, -1, -1, -1, -1, 3},   // 241
    { 0,  8, 10,  0, 10, 11,  0, 11,  5, -1, -1, -1, -1, -1, -1, 3},   // 242
    { 4, 10, 11,  4, 11,  5, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 243
    { 1, 11,  9,  1,  9,  8,  1,  8,  4, -1, -1, -1, -1, -1, -1, 3},   // 244
    { 0,  1, 11,  0, 11,  9, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 245
    { 8,  4,  1,  8,  1, 11,  8, 11,  5,  8,  5,  0, -1, -1, -1, 4},   // 246
    { 1, 11,  5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   // 247
    { 1,  5,  9,  1,  9,  8,  1,  8, 10, -1, -1, -1, -1, -1, -1, 3},   // 248
    {10,  1,  5, 10,  5,  9, 10,  9,  0, 10,  0,  4, -1, -1, -1, 4},   // 249
    { 0,  8, 10,  0, 10,  1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 250
    { 1,  4, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   // 251
    { 4,  5,  9,  4,  9,  8, -1, -1, -1, -1, -1, -1, -1, -1, -1, 2},   // 252
    { 0,  5,  9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   // 253
    { 0,  8,  4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 1},   // 254
    {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 0},   // 255
};

struct Geom {
    const float* g;
    int nz, ny, nx;
    float level;
    int rows;             // nz * ny
    int tiles;            // scan tiles
    int64_t* ws;          // [3][rows] row sums, scanned in place into offsets; then [3][tiles] tile sums
};

__device__ __forceinline__ const float* row_ptr(const Geom& p, int b0, int b1) { return p.g + ((int64_t)b0 * p.ny + b1) * p.nx; }

// The lane's voxel a2 of row (b0, b1) and the voxel after it (0 past the row, and for a row outside the grid).  All lanes call it.
__device__ __forceinline__ void load_pair(const Geom& p, int b0, int b1, int a2, int lane, float& v, float& vn) {
    const bool row = b0 < p.nz && b1 < p.ny;
    const float* r = row ? row_ptr(p, b0, b1) : nullptr;
    v = row && a2 < p.nx ? __ldg(r + a2) : 0.f;
    vn = __shfl_down_sync(0xffffffffu, v, 1);
    if (lane == 31) vn = row && a2 + 1 < p.nx ? __ldg(r + a2 + 1) : 0.f;
}

// Crossed x / y / z edges (bits 0 / 1 / 2) of voxel a2 of row (b0, b1), from its value v, the next voxel vn, and the voxels vy
// at b1 + 1 and vz at b0 + 1.  A grid with a dimension below 2 has no cells and no vertices.
__device__ __forceinline__ int edge_bits(const Geom& p, int b0, int b1, int a2, float v, float vn, float vy, float vz) {
    if (b0 >= p.nz || b1 >= p.ny || a2 >= p.nx || p.nz < 2 || p.ny < 2 || p.nx < 2) return 0;
    const bool in = v > p.level;
    return (a2 + 1 < p.nx && in != (vn > p.level)) | (b1 + 1 < p.ny && in != (vy > p.level)) << 1 |
           (b0 + 1 < p.nz && in != (vz > p.level)) << 2;
}

__device__ __forceinline__ int config(float level, float c0, float c1, float c2, float c3, float c4, float c5, float c6, float c7) {
    return (c0 > level) | (c1 > level) << 1 | (c2 > level) << 2 | (c3 > level) << 3 | (c4 > level) << 4 | (c5 > level) << 5 |
           (c6 > level) << 6 | (c7 > level) << 7;
}

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ int warp_inclusive(int v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    return v;
}

__global__ void __launch_bounds__(32 * kWarps) iso_count_rows(Geom p) {
    const int lane = threadIdx.x & 31;
    const bool cells = p.nz > 1 && p.ny > 1 && p.nx > 1;
    for (int r = blockIdx.x * kWarps + (threadIdx.x >> 5); r < p.rows; r += gridDim.x * kWarps) {
        const int a0 = r / p.ny, a1 = r - a0 * p.ny;
        const bool cell_row = cells && a0 + 1 < p.nz && a1 + 1 < p.ny;
        int nv = 0, nt = 0, nf = 0;
        for (int base = 0; base < p.nx; base += 32) {
            const int a2 = base + lane;
            float v0, v0n, v1, v1n, v2, v2n, v3, v3n;
            load_pair(p, a0, a1, a2, lane, v0, v0n);
            load_pair(p, a0, a1 + 1, a2, lane, v1, v1n);
            load_pair(p, a0 + 1, a1, a2, lane, v2, v2n);
            load_pair(p, a0 + 1, a1 + 1, a2, lane, v3, v3n);
            nf += a2 < p.nx && !isfinite(v0);
            nv += __popc(edge_bits(p, a0, a1, a2, v0, v0n, v1, v2));
            if (cell_row && a2 + 1 < p.nx) nt += c_tri[config(p.level, v0, v0n, v1, v1n, v2, v2n, v3, v3n)][15];
        }
        nv = warp_sum(nv);
        nt = warp_sum(nt);
        nf = warp_sum(nf);
        if (lane == 0) {
            p.ws[r] = nv;
            p.ws[p.rows + r] = nt;
            p.ws[2 * (int64_t)p.rows + r] = nf;
        }
    }
}

// Exclusive scan of one value per thread over the block (kScanThreads threads); *total receives the block's sum.
__device__ int64_t block_exclusive(int64_t v, int64_t* total) {
    __shared__ int64_t s_warp[kScanThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
    }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    if (w == 0) {
        int64_t s = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t u = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += u;
        }
        s_warp[lane] = s;
    }
    __syncthreads();
    const int64_t out = (w ? s_warp[w - 1] : 0) + inc - v;
    *total = s_warp[kScanThreads / 32 - 1];
    __syncthreads();
    return out;
}

__global__ void __launch_bounds__(kScanThreads) iso_scan_tiles(Geom p) {
    int64_t* tile = p.ws + 3 * (int64_t)p.rows;
    for (int k = 0; k < 3; ++k) {
        const int64_t* a = p.ws + k * (int64_t)p.rows;
        int64_t s = 0;
        for (int i = 0; i < kTile / kScanThreads; ++i) {
            const int64_t r = (int64_t)blockIdx.x * kTile + i * kScanThreads + threadIdx.x;
            if (r < p.rows) s += a[r];
        }
        int64_t total;
        block_exclusive(s, &total);
        if (threadIdx.x == 0) tile[k * p.tiles + blockIdx.x] = total;
    }
}

__global__ void __launch_bounds__(kScanThreads) iso_scan_rows(Geom p, int64_t* counts) {
    const int64_t* tile = p.ws + 3 * (int64_t)p.rows;
    for (int k = 0; k < 3; ++k) {
        int64_t before = 0, total;
        for (int t = threadIdx.x; t < (int)blockIdx.x; t += kScanThreads) before += tile[k * p.tiles + t];
        block_exclusive(before, &total);
        before = total;
        int64_t* a = p.ws + k * (int64_t)p.rows;
        const int64_t r0 = (int64_t)blockIdx.x * kTile + 4 * threadIdx.x;      // four consecutive rows per thread
        int64_t v[4], s = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            v[i] = r0 + i < p.rows ? a[r0 + i] : 0;
            s += v[i];
        }
        int64_t off = before + block_exclusive(s, &total);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (r0 + i < p.rows) a[r0 + i] = off;
            off += v[i];
        }
        if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) counts[k] = before + total;
    }
}

struct RowIds {           // one row's vertex ids at the lane's voxel: id of its x-, y- and z-edge vertex (if crossed)
    int x, y, z;
};

// In-row prefix of row (b0, b1) (vertex offset `off`, running count `carry` of the voxels before this chunk): the lane's ids.
__device__ __forceinline__ RowIds row_ids(int bits, int64_t off, int& carry, int lane) {
    const int n = __popc(bits), inc = warp_inclusive(n, lane);
    const int x = (int)(off + carry + inc - n);
    carry += __shfl_sync(0xffffffffu, inc, 30);          // lanes 0..30 own this chunk's voxels; lane 31's is the next chunk's first
    return {x, x + (bits & 1), x + (bits & 1) + (bits >> 1 & 1)};
}

__global__ void __launch_bounds__(32 * kWarps) iso_emit_rows(Geom p, float* __restrict__ verts, int32_t* __restrict__ faces) {
    __shared__ int s_id[kWarps][12][32];     // the lane's cell: vertex id of each of its 12 edges
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const bool cells = p.nz > 1 && p.ny > 1 && p.nx > 1;
    if (!cells) return;
    const int64_t* voff = p.ws;
    const int64_t* toff = p.ws + p.rows;
    for (int r = blockIdx.x * kWarps + w; r < p.rows; r += gridDim.x * kWarps) {
        const int a0 = r / p.ny, a1 = r - a0 * p.ny;
        const bool cell_row = a0 + 1 < p.nz && a1 + 1 < p.ny;
        // rows (a0 + i, a1 + j) = rij; a cell row needs the vertices of r00, r01, r10 and r11
        const int64_t o00 = voff[r];
        const int64_t o01 = cell_row ? voff[r + 1] : 0, o10 = cell_row ? voff[r + p.ny] : 0, o11 = cell_row ? voff[r + p.ny + 1] : 0;
        const int64_t t0 = cell_row ? toff[r] : 0;
        int c00 = 0, c01 = 0, c10 = 0, c11 = 0, ct = 0;
        for (int base = 0; base < p.nx; base += 31) {
            const int a2 = base + lane;
            float v00, n00, v01, n01, v10, n10, v11, n11, v02, n02, v20, n20, v12, n12, v21, n21;
            load_pair(p, a0, a1, a2, lane, v00, n00);
            load_pair(p, a0, a1 + 1, a2, lane, v01, n01);
            load_pair(p, a0 + 1, a1, a2, lane, v10, n10);
            const int b00 = edge_bits(p, a0, a1, a2, v00, n00, v01, v10);
            const RowIds i00 = row_ids(b00, o00, c00, lane);
            if (lane < 31 && b00) {
                const float x = (float)a2, y = (float)a1, z = (float)a0;
                if (b00 & 1) {
                    float* o = verts + 3 * (int64_t)i00.x;
                    o[0] = __fadd_rn(x, __fdiv_rn(__fsub_rn(p.level, v00), __fsub_rn(n00, v00)));
                    o[1] = y;
                    o[2] = z;
                }
                if (b00 & 2) {
                    float* o = verts + 3 * (int64_t)i00.y;
                    o[0] = x;
                    o[1] = __fadd_rn(y, __fdiv_rn(__fsub_rn(p.level, v00), __fsub_rn(v01, v00)));
                    o[2] = z;
                }
                if (b00 & 4) {
                    float* o = verts + 3 * (int64_t)i00.z;
                    o[0] = x;
                    o[1] = y;
                    o[2] = __fadd_rn(z, __fdiv_rn(__fsub_rn(p.level, v00), __fsub_rn(v10, v00)));
                }
            }
            if (!cell_row) continue;
            load_pair(p, a0 + 1, a1 + 1, a2, lane, v11, n11);
            load_pair(p, a0, a1 + 2, a2, lane, v02, n02);
            load_pair(p, a0 + 2, a1, a2, lane, v20, n20);
            load_pair(p, a0 + 1, a1 + 2, a2, lane, v12, n12);
            load_pair(p, a0 + 2, a1 + 1, a2, lane, v21, n21);
            const RowIds i01 = row_ids(edge_bits(p, a0, a1 + 1, a2, v01, n01, v02, v11), o01, c01, lane);
            const RowIds i10 = row_ids(edge_bits(p, a0 + 1, a1, a2, v10, n10, v11, v20), o10, c10, lane);
            const RowIds i11 = row_ids(edge_bits(p, a0 + 1, a1 + 1, a2, v11, n11, v12, v21), o11, c11, lane);
            const int cfg = config(p.level, v00, n00, v01, n01, v10, n10, v11, n11);
            const int4 e = *reinterpret_cast<const int4*>(c_tri[cfg]);
            const int nt = lane < 31 && a2 + 1 < p.nx ? (e.w >> 24) : 0;
            const int inc = warp_inclusive(nt, lane);
            const int64_t first = t0 + ct + inc - nt;
            ct += __shfl_sync(0xffffffffu, inc, 31);
            int* id = &s_id[w][0][lane];
            id[0 * 32] = i00.x;
            id[1 * 32] = i01.x;
            id[2 * 32] = i10.x;
            id[3 * 32] = i11.x;
            id[4 * 32] = i00.y;
            id[5 * 32] = __shfl_down_sync(0xffffffffu, i00.y, 1);
            id[6 * 32] = i10.y;
            id[7 * 32] = __shfl_down_sync(0xffffffffu, i10.y, 1);
            id[8 * 32] = i00.z;
            id[9 * 32] = __shfl_down_sync(0xffffffffu, i00.z, 1);
            id[10 * 32] = i01.z;
            id[11 * 32] = __shfl_down_sync(0xffffffffu, i01.z, 1);
            const int words[4] = {e.x, e.y, e.z, e.w};
#pragma unroll
            for (int j = 0; j < 15; ++j) {
                if (j < 3 * nt) faces[3 * first + j] = id[(int8_t)(words[j >> 2] >> (8 * (j & 3))) * 32];
            }
        }
    }
}

int make_geom(const float* grid, int nz, int ny, int nx, float level, void* workspace, Geom& p, const char* who) {
    N3D_CHECK_ARG(nz > 0 && ny > 0 && nx > 0, "%s: need nz, ny, nx > 0, got %d, %d, %d", who, nz, ny, nx);
    N3D_CHECK_ARG((int64_t)nz * ny <= 0x7fffffffLL - kTile && nx <= (1 << 28), "%s: a %dx%dx%d grid is too large", who, nz, ny, nx);
    N3D_CHECK_ARG(isfinite(level), "%s: the level must be finite", who);
    p.g = grid;
    p.nz = nz;
    p.ny = ny;
    p.nx = nx;
    p.level = level;
    p.rows = nz * ny;
    p.tiles = n3d_div_up(p.rows, kTile);
    p.ws = (int64_t*)workspace;
    return N3D_OK;
}

}  // namespace

extern "C" int n3d_isosurface_workspace_bytes(int nz, int ny, int nx, size_t* bytes) {
    N3D_CHECK_ARG(bytes, "n3d_isosurface_workspace_bytes: null output pointer");
    Geom p;
    const int rc = make_geom(nullptr, nz, ny, nx, 0.f, nullptr, p, "n3d_isosurface_workspace_bytes");
    if (rc != N3D_OK) return rc;
    *bytes = 3 * sizeof(int64_t) * ((size_t)p.rows + p.tiles);
    return N3D_OK;
}

extern "C" int n3d_isosurface_count(const float* grid, int nz, int ny, int nx, float level, void* workspace, int64_t* counts,
                                    void* stream) {
    N3D_CHECK_ARG(grid && workspace && counts, "n3d_isosurface_count: null buffer");
    N3D_CHECK_ARG((uintptr_t)workspace % 8 == 0, "n3d_isosurface_count: the workspace must be 8-byte aligned");
    Geom p;
    const int rc = make_geom(grid, nz, ny, nx, level, workspace, p, "n3d_isosurface_count");
    if (rc != N3D_OK) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    iso_count_rows<<<n3d_grid((int64_t)p.rows * 32, 32 * kWarps), 32 * kWarps, 0, s>>>(p);
    iso_scan_tiles<<<p.tiles, kScanThreads, 0, s>>>(p);
    iso_scan_rows<<<p.tiles, kScanThreads, 0, s>>>(p, counts);
    N3D_CHECK_LAUNCH("n3d_isosurface_count");
    return N3D_OK;
}

extern "C" int n3d_isosurface_emit(const float* grid, int nz, int ny, int nx, float level, const void* workspace, float* verts,
                                   int32_t* faces, void* stream) {
    N3D_CHECK_ARG(grid && workspace && verts && faces, "n3d_isosurface_emit: null buffer");
    N3D_CHECK_ARG((uintptr_t)workspace % 8 == 0, "n3d_isosurface_emit: the workspace must be 8-byte aligned");
    Geom p;
    const int rc = make_geom(grid, nz, ny, nx, level, (void*)workspace, p, "n3d_isosurface_emit");
    if (rc != N3D_OK) return rc;
    iso_emit_rows<<<n3d_grid((int64_t)p.rows * 32, 32 * kWarps), 32 * kWarps, 0, (cudaStream_t)stream>>>(p, verts, faces);
    N3D_CHECK_LAUNCH("n3d_isosurface_emit");
    return N3D_OK;
}
