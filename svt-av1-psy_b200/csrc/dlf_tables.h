/* dlf_tables.h -- the small AV1 tables the deblocking edge derivation reads, as initialiser lists shared by the device
 * code (dlf.cu puts them in __constant__ memory) and by plain C (the CPU checker compares them with the reference's).
 *
 * Indices follow the AV1 enumerations: BlockSize (22 values: 4X4, 4X8, 8X4, 8X8, 8X16, 16X8, 16X16, 16X32, 32X16, 32X32,
 * 32X64, 64X32, 64X64, 64X128, 128X64, 128X128, 4X16, 16X4, 8X32, 32X8, 16X64, 64X16), TxSize (19 values: 4X4, 8X8,
 * 16X16, 32X32, 64X64, 4X8, 8X4, 8X16, 16X8, 16X32, 32X16, 32X64, 64X32, 4X16, 16X4, 8X32, 32X8, 16X64, 64X16) and
 * PredictionMode (25 values: 13 intra modes, NEARESTMV, NEARMV, GLOBALMV, NEWMV, then the 8 compound modes). */
#ifndef SVT_B200_DLF_TABLES_H
#define SVT_B200_DLF_TABLES_H

#define B200_DLF_N_BSIZE 22
#define B200_DLF_N_TXSIZE 19
#define B200_DLF_N_MODES 25

/* Luma transform size of a block coded at transform depth 0, 1, 2: the largest rectangular transform that fits the block
 * (at most 64 on a side), split `depth` times (a square splits into four squares, a 2:1 rectangle into two squares, a
 * 4:1 rectangle into two 2:1 rectangles).  A depth the block does not allow keeps the depth-0 size: 4X4, 4X8, 8X4 and
 * the 128 sizes at depths 1 and 2, 8X8 at depth 2. */
#define B200_DLF_TX_DEPTH_TO_TX_SIZE                                                                                    \
    {{0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 11, 12, 4, 4, 4, 4, 13, 14, 15, 16, 17, 18},                                      \
     {0, 5, 6, 0, 1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4, 5, 6, 7, 8, 9, 10},                                             \
     {0, 5, 6, 1, 0, 0, 0, 1, 1, 1, 2, 2, 2, 4, 4, 4, 0, 0, 1, 1, 2, 2}}

/* Chroma transform size of a block in 4:2:0: the largest transform of the subsampled block, with 64-point sizes reduced
 * to 32 (a chroma block never uses a 64-point transform). */
#define B200_DLF_UV_TX_SIZE_420 {0, 0, 0, 0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 3, 3, 3, 5, 6, 13, 14, 15, 16}

/* The square transform size that has a transform's width (horz) resp. height (vert). */
#define B200_DLF_TXSIZE_HORZ_MAP {0, 1, 2, 3, 4, 0, 1, 1, 2, 2, 3, 3, 4, 0, 2, 1, 3, 2, 4}
#define B200_DLF_TXSIZE_VERT_MAP {0, 1, 2, 3, 4, 1, 0, 2, 1, 3, 2, 4, 3, 2, 0, 3, 1, 4, 2}

/* Block size of a block's chroma in 4:2:0 (both dimensions halved, at least 4). */
#define B200_DLF_PLANE_BSIZE_420 {0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 1, 2, 16, 17, 18, 19}

/* Block width / height in pixels. */
#define B200_DLF_BLOCK_W {4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 64, 128, 128, 4, 16, 8, 32, 16, 64}
#define B200_DLF_BLOCK_H {4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 64, 32, 64, 128, 64, 128, 16, 4, 32, 8, 64, 16}

/* Which of the two mode deltas of a frame's loop-filter header a prediction mode takes: 1 for inter modes that code a
 * motion vector, 0 for intra modes and the global-motion modes GLOBALMV and GLOBAL_GLOBALMV. */
#define B200_DLF_MODE_LF_LUT {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, 0, 1}

#endif /* SVT_B200_DLF_TABLES_H */
