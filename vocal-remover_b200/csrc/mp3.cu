// MPEG-1 Audio Layer III decoding (ISO/IEC 11172-3) on the device: the decode in front of the hot path for .mp3 input
// (lib/mp3.py drives it; oracle/mp3_oracle.py restates the standard in float64 and is pinned against FFmpeg).
//
// No stage loops over granules: every dependency between granules is recomputed or left to a later kernel.
//   mp3_scan_kernel       one thread per byte: every 11-bit sync with its 4 header bytes (warp-aggregated appends);
//                         the host walks the frame chain and takes the exclusive scan of the main-data byte counts.
//   mp3_side_info_kernel  one thread per frame: header and side info -> one descriptor per granule-channel with the
//                         bit offset of its part2_3 data in the reservoir buffer (the frame's main-data offset less
//                         main_data_begin, plus the lengths before it in the frame); status per frame.
//   mp3_gather_kernel     one CTA per frame: main data to its offset in one contiguous reservoir buffer.
//   mp3_huffman_kernel    one thread per granule-channel: scale factors (a granule 1 that shares groups by scfsi
//                         re-reads granule 0's bits at their known offset), Huffman decoding with the tables in shared
//                         memory (a binary search over each table's left-aligned codes), requantisation with
//                         |x|^(4/3) from a table.  Every read is bounded by the granule and the buffer; a malformed
//                         granule leaves code << 40 | bit offset and decodes as zeros.
//   mp3_stereo_kernel     one thread per joint-stereo granule: MS, and MPEG-1 intensity stereo over the right
//                         channel's zero part.
//   mp3_hybrid_kernel     one CTA per granule-channel: short-block reorder, antialias butterflies, IMDCT of this
//                         granule and of the previous one (its tail is recomputed, not carried), overlap-add, frequency
//                         inversion, and the 64-value V vector of each of the 18 subband slots.
//   mp3_window_kernel     one thread per output sample: the 512-tap window D over the 16 V vectors up to its slot.
#include <math.h>

#include "bitstream.cuh"
#include "common.cuh"
#include "kernels.h"

namespace vr {

namespace {

// Huffman code tables 1 2 3 5 6 7 8 9 10 11 12 13 15 16 24 as symbols (x << 4 | y) and code lengths in increasing code
// order (oracle/mp3_tables.py states the convention); the synthesis window D[0..256] times 65536.
__constant__ uint8_t kHuffSymbols[1378] = {
    17, 1, 16, 0, 34, 2, 18, 33, 32, 17, 1, 16, 0, 34, 2, 18, 33, 32, 16, 17, 1, 0, 51, 35, 50, 49, 19, 3, 48, 34,
    18, 33, 2, 32, 17, 1, 16, 0, 51, 3, 35, 50, 48, 19, 49, 34, 2, 18, 33, 32, 1, 17, 16, 0, 85, 69, 84, 83, 53, 68,
    37, 82, 21, 81, 5, 52, 80, 67, 51, 36, 66, 20, 65, 64, 4, 35, 50, 3, 19, 49, 48, 34, 18, 33, 2, 32, 17, 1, 16,
    0, 85, 84, 69, 83, 53, 68, 37, 82, 5, 21, 81, 52, 67, 80, 51, 36, 66, 20, 65, 4, 64, 35, 50, 19, 49, 3, 48, 34,
    2, 32, 18, 33, 17, 1, 16, 0, 85, 69, 53, 83, 84, 5, 68, 37, 82, 21, 81, 52, 67, 80, 4, 36, 66, 51, 64, 20, 65,
    35, 50, 19, 49, 3, 48, 34, 2, 18, 33, 32, 17, 1, 16, 0, 119, 103, 118, 87, 117, 102, 71, 116, 86, 101, 55, 115,
    70, 85, 84, 99, 39, 114, 100, 7, 112, 98, 69, 53, 6, 83, 68, 23, 113, 54, 38, 37, 82, 21, 81, 52, 67, 22, 97,
    96, 5, 80, 36, 66, 51, 4, 20, 65, 64, 35, 50, 3, 19, 49, 48, 34, 18, 33, 2, 32, 17, 1, 16, 0, 119, 103, 118,
    117, 102, 71, 116, 87, 85, 86, 101, 55, 115, 70, 69, 84, 53, 83, 39, 114, 100, 7, 113, 23, 112, 54, 99, 96, 68,
    37, 82, 5, 21, 98, 38, 6, 22, 97, 81, 52, 80, 67, 51, 36, 66, 20, 65, 4, 64, 35, 50, 19, 49, 3, 48, 34, 33, 18,
    2, 32, 17, 1, 16, 0, 119, 103, 118, 87, 117, 102, 71, 116, 101, 86, 55, 115, 85, 39, 114, 70, 100, 23, 113, 7,
    112, 54, 99, 69, 84, 68, 6, 5, 38, 98, 97, 22, 96, 53, 83, 37, 82, 21, 81, 52, 67, 80, 4, 36, 66, 20, 51, 65,
    35, 50, 64, 3, 48, 19, 49, 34, 18, 33, 2, 32, 0, 17, 1, 16, 254, 252, 253, 237, 255, 239, 223, 238, 207, 222,
    191, 251, 206, 220, 175, 233, 236, 221, 250, 205, 190, 235, 159, 249, 234, 189, 219, 143, 248, 204, 174, 158,
    142, 127, 126, 247, 218, 173, 188, 203, 246, 111, 232, 95, 157, 217, 245, 231, 172, 187, 79, 244, 202, 230, 243,
    63, 141, 216, 47, 242, 110, 156, 15, 201, 94, 171, 125, 215, 78, 200, 214, 62, 185, 155, 170, 31, 241, 240, 186,
    229, 228, 140, 109, 227, 226, 46, 14, 30, 225, 224, 93, 213, 124, 199, 77, 139, 184, 212, 154, 169, 108, 198,
    61, 211, 123, 45, 210, 29, 183, 92, 197, 153, 122, 195, 167, 151, 75, 209, 13, 208, 138, 168, 76, 196, 107, 182,
    60, 44, 194, 91, 181, 137, 28, 193, 152, 12, 192, 180, 106, 166, 121, 59, 179, 136, 90, 43, 165, 105, 164, 120,
    135, 148, 119, 118, 178, 27, 177, 11, 176, 150, 74, 58, 163, 89, 149, 42, 162, 26, 161, 10, 104, 160, 134, 73,
    147, 57, 88, 133, 103, 41, 146, 87, 117, 56, 131, 102, 71, 116, 86, 101, 115, 25, 145, 9, 144, 72, 132, 114, 70,
    100, 40, 130, 24, 55, 39, 23, 113, 85, 7, 112, 54, 99, 69, 84, 38, 98, 53, 129, 8, 128, 22, 97, 6, 96, 83, 68,
    37, 82, 5, 21, 81, 52, 67, 80, 36, 66, 51, 20, 65, 4, 64, 35, 50, 19, 49, 3, 48, 34, 18, 33, 2, 32, 17, 1, 16,
    0, 255, 239, 254, 223, 238, 253, 207, 252, 222, 237, 191, 251, 206, 236, 221, 175, 250, 190, 235, 205, 220, 159,
    249, 234, 189, 219, 143, 248, 204, 158, 233, 127, 247, 173, 218, 188, 111, 174, 15, 203, 246, 142, 232, 95, 157,
    245, 126, 231, 172, 202, 187, 217, 141, 79, 244, 63, 243, 216, 230, 47, 242, 110, 240, 31, 241, 156, 201, 94,
    171, 186, 229, 125, 215, 78, 228, 140, 200, 62, 109, 214, 227, 155, 185, 46, 170, 226, 30, 225, 14, 224, 93,
    213, 124, 199, 77, 139, 212, 184, 154, 169, 108, 198, 61, 211, 210, 45, 13, 29, 123, 183, 209, 92, 208, 197,
    138, 168, 76, 196, 107, 182, 153, 12, 60, 195, 122, 167, 166, 192, 11, 194, 44, 91, 181, 28, 137, 152, 193, 75,
    180, 106, 59, 121, 179, 151, 136, 43, 90, 178, 165, 27, 177, 176, 105, 150, 74, 164, 120, 135, 58, 163, 89, 149,
    42, 162, 26, 161, 10, 160, 104, 134, 73, 148, 57, 147, 119, 9, 88, 133, 41, 103, 118, 146, 145, 25, 144, 72,
    132, 87, 117, 56, 131, 102, 71, 40, 130, 24, 129, 116, 8, 128, 86, 101, 55, 115, 70, 39, 114, 100, 23, 85, 113,
    7, 112, 54, 99, 69, 84, 38, 98, 22, 6, 96, 53, 97, 83, 68, 37, 82, 21, 81, 5, 80, 52, 67, 36, 66, 51, 65, 20, 4,
    35, 50, 64, 3, 19, 49, 48, 34, 18, 33, 2, 32, 17, 1, 16, 0, 239, 254, 223, 253, 207, 252, 191, 251, 175, 250,
    159, 249, 248, 143, 127, 247, 111, 246, 255, 95, 245, 79, 244, 243, 240, 63, 206, 236, 221, 222, 233, 234, 217,
    238, 237, 235, 190, 205, 220, 219, 174, 204, 173, 218, 126, 172, 202, 201, 125, 94, 189, 242, 47, 15, 31, 241,
    158, 188, 203, 142, 232, 157, 231, 187, 141, 216, 110, 230, 156, 171, 186, 229, 215, 78, 228, 140, 200, 62, 109,
    214, 155, 185, 170, 225, 212, 184, 169, 123, 183, 208, 227, 14, 224, 93, 213, 124, 199, 77, 139, 154, 108, 198,
    61, 92, 197, 13, 138, 168, 153, 76, 182, 122, 60, 91, 137, 28, 192, 152, 121, 226, 46, 30, 211, 45, 210, 209,
    59, 151, 136, 29, 196, 107, 195, 167, 44, 194, 181, 193, 12, 75, 180, 106, 166, 179, 90, 165, 43, 178, 27, 177,
    11, 176, 105, 150, 74, 164, 120, 135, 163, 58, 89, 42, 149, 104, 161, 134, 119, 148, 73, 87, 103, 162, 26, 10,
    160, 57, 147, 88, 133, 41, 146, 118, 9, 25, 145, 144, 72, 132, 117, 56, 131, 102, 40, 130, 71, 116, 24, 129,
    128, 8, 86, 55, 115, 101, 70, 39, 114, 100, 85, 7, 23, 113, 112, 54, 99, 69, 84, 38, 98, 22, 97, 6, 96, 83, 53,
    68, 37, 82, 81, 21, 5, 52, 67, 80, 36, 66, 51, 20, 65, 4, 64, 35, 50, 19, 49, 3, 48, 34, 18, 33, 2, 32, 17, 1,
    16, 0, 239, 254, 223, 253, 207, 252, 191, 251, 250, 175, 159, 249, 248, 143, 127, 247, 111, 246, 95, 245, 79,
    244, 63, 243, 47, 242, 241, 31, 240, 15, 238, 222, 237, 206, 236, 221, 190, 235, 205, 220, 174, 234, 189, 219,
    204, 158, 233, 173, 218, 188, 203, 142, 232, 157, 217, 126, 231, 172, 255, 202, 187, 141, 216, 14, 224, 13, 230,
    110, 156, 201, 94, 186, 229, 171, 125, 215, 228, 140, 200, 78, 46, 62, 109, 214, 227, 155, 185, 170, 226, 30,
    225, 93, 213, 124, 199, 77, 139, 184, 212, 154, 169, 108, 198, 61, 211, 45, 210, 29, 123, 183, 209, 92, 197,
    138, 168, 153, 76, 196, 107, 182, 208, 12, 60, 195, 122, 167, 44, 194, 91, 181, 28, 137, 152, 193, 75, 192, 11,
    59, 176, 10, 26, 180, 106, 166, 121, 151, 160, 9, 144, 179, 136, 43, 90, 178, 165, 27, 177, 105, 150, 164, 74,
    120, 135, 58, 163, 89, 149, 42, 162, 161, 104, 134, 119, 73, 148, 57, 147, 88, 133, 41, 103, 118, 146, 25, 145,
    72, 132, 87, 117, 56, 131, 102, 40, 130, 24, 71, 116, 129, 8, 128, 86, 101, 23, 7, 112, 115, 55, 39, 114, 70,
    100, 85, 113, 54, 99, 69, 84, 38, 98, 22, 97, 6, 96, 53, 83, 68, 37, 82, 21, 5, 80, 81, 52, 67, 36, 66, 51, 20,
    65, 4, 64, 35, 50, 19, 49, 3, 48, 34, 18, 33, 2, 32, 17, 1, 16, 0};

__constant__ uint8_t kHuffLengths[1378] = {
    3, 3, 2, 1, 6, 6, 5, 5, 5, 3, 3, 3, 1, 6, 6, 5, 5, 5, 3, 2, 2, 2, 8, 8, 7, 6, 7, 7, 7, 7, 6, 6, 6, 6, 3, 3, 3,
    1, 7, 7, 6, 6, 6, 5, 5, 5, 5, 4, 4, 4, 3, 2, 3, 3, 10, 10, 10, 10, 9, 9, 9, 9, 8, 8, 9, 9, 8, 9, 9, 8, 8, 7, 7,
    7, 8, 8, 8, 8, 7, 7, 7, 7, 6, 5, 6, 6, 4, 3, 3, 1, 11, 11, 10, 9, 10, 10, 9, 9, 9, 8, 8, 9, 9, 9, 9, 8, 8, 8, 7,
    8, 8, 8, 8, 8, 8, 8, 8, 6, 6, 6, 4, 4, 2, 3, 3, 2, 9, 9, 8, 8, 9, 9, 8, 8, 8, 8, 7, 7, 7, 8, 8, 7, 7, 7, 7, 6,
    6, 6, 6, 5, 5, 6, 6, 5, 5, 4, 4, 4, 3, 3, 3, 3, 11, 11, 11, 11, 11, 11, 10, 10, 10, 10, 10, 10, 10, 11, 11, 10,
    9, 9, 10, 10, 9, 9, 10, 10, 9, 10, 10, 8, 8, 9, 9, 10, 10, 9, 9, 10, 10, 8, 8, 8, 9, 9, 9, 9, 9, 9, 8, 8, 8, 8,
    8, 8, 7, 7, 7, 7, 6, 6, 6, 6, 4, 3, 3, 1, 10, 10, 10, 10, 10, 10, 10, 11, 11, 10, 10, 9, 9, 9, 10, 10, 10, 10,
    8, 8, 9, 9, 7, 8, 8, 8, 8, 8, 9, 9, 9, 9, 8, 7, 8, 8, 7, 7, 8, 8, 8, 9, 9, 8, 8, 8, 8, 8, 8, 7, 7, 6, 6, 7, 7,
    6, 5, 4, 5, 5, 3, 3, 3, 2, 10, 10, 9, 9, 9, 9, 9, 9, 9, 8, 8, 9, 9, 8, 8, 8, 8, 8, 8, 9, 9, 8, 8, 8, 8, 8, 9, 9,
    7, 7, 7, 8, 8, 8, 8, 8, 8, 7, 7, 7, 7, 8, 8, 7, 7, 7, 6, 6, 6, 6, 7, 7, 6, 5, 5, 5, 4, 4, 5, 5, 4, 3, 3, 3, 19,
    19, 18, 17, 16, 16, 16, 16, 16, 16, 16, 16, 16, 16, 17, 17, 15, 15, 16, 16, 15, 15, 15, 15, 15, 15, 15, 15, 15,
    15, 16, 16, 15, 16, 16, 14, 14, 15, 15, 15, 15, 14, 14, 14, 14, 14, 14, 14, 14, 14, 14, 14, 15, 15, 14, 13, 14,
    14, 13, 13, 14, 14, 13, 14, 14, 13, 14, 14, 13, 14, 14, 13, 13, 14, 14, 12, 12, 12, 13, 13, 13, 13, 13, 13, 12,
    13, 13, 12, 12, 13, 13, 13, 13, 13, 13, 13, 13, 13, 13, 13, 13, 12, 12, 13, 13, 12, 12, 12, 12, 13, 13, 13, 13,
    12, 13, 13, 12, 11, 12, 12, 12, 12, 12, 12, 12, 12, 11, 11, 11, 11, 12, 12, 11, 11, 12, 12, 11, 12, 12, 12, 12,
    11, 11, 12, 12, 11, 12, 12, 11, 12, 12, 11, 12, 12, 10, 10, 10, 11, 11, 11, 11, 11, 11, 11, 11, 10, 10, 10, 10,
    11, 11, 10, 11, 11, 10, 11, 11, 11, 11, 10, 10, 11, 11, 10, 10, 11, 11, 11, 11, 11, 11, 9, 9, 10, 10, 10, 10,
    10, 11, 11, 9, 9, 9, 10, 10, 9, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 8, 9, 9, 9, 9, 9, 9, 10, 10, 9, 9, 9,
    8, 8, 9, 9, 9, 9, 9, 9, 8, 7, 8, 8, 8, 8, 7, 7, 7, 7, 7, 6, 6, 6, 6, 4, 4, 3, 1, 13, 13, 13, 13, 12, 13, 13, 13,
    13, 13, 13, 12, 13, 13, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12, 12,
    12, 13, 13, 11, 11, 12, 12, 12, 12, 11, 11, 11, 11, 11, 11, 12, 12, 11, 11, 11, 11, 11, 11, 11, 11, 12, 12, 11,
    11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 12, 12, 11, 11,
    11, 11, 11, 11, 10, 11, 11, 11, 11, 11, 11, 10, 10, 11, 11, 10, 10, 10, 10, 11, 11, 10, 10, 10, 10, 10, 10, 10,
    11, 11, 10, 10, 10, 10, 10, 11, 11, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 9, 10, 10, 10, 10, 9, 10,
    10, 9, 10, 10, 10, 10, 10, 10, 10, 10, 9, 9, 9, 9, 9, 9, 9, 10, 10, 9, 9, 9, 9, 9, 9, 10, 10, 9, 9, 9, 9, 9, 9,
    8, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 8, 8, 8, 8, 9, 9, 9, 9, 9, 9, 9, 9, 8, 8, 8, 8, 8, 8, 9, 9, 8, 8, 8, 8, 8, 8,
    8, 9, 9, 8, 7, 8, 8, 7, 7, 7, 7, 8, 8, 7, 7, 7, 7, 7, 6, 7, 7, 6, 6, 7, 7, 6, 6, 6, 5, 5, 5, 5, 5, 3, 4, 4, 3,
    11, 11, 11, 11, 11, 11, 11, 11, 10, 11, 11, 11, 11, 10, 10, 10, 10, 10, 8, 10, 10, 9, 9, 9, 9, 10, 16, 17, 17,
    15, 15, 16, 16, 14, 15, 15, 14, 14, 15, 15, 14, 14, 15, 15, 15, 15, 14, 15, 15, 14, 13, 8, 9, 9, 8, 8, 13, 14,
    14, 14, 14, 14, 14, 14, 14, 14, 14, 13, 13, 14, 14, 14, 14, 13, 14, 14, 13, 13, 13, 14, 14, 14, 14, 13, 13, 14,
    14, 13, 14, 14, 12, 13, 13, 13, 13, 13, 13, 13, 13, 13, 13, 13, 13, 13, 13, 12, 13, 13, 13, 13, 13, 13, 12, 13,
    13, 12, 12, 13, 13, 11, 12, 12, 12, 12, 12, 12, 12, 13, 13, 11, 12, 12, 12, 12, 11, 12, 12, 12, 12, 12, 12, 12,
    12, 11, 12, 12, 11, 11, 11, 11, 12, 12, 12, 12, 12, 12, 12, 12, 11, 12, 12, 11, 12, 12, 11, 12, 12, 11, 12, 12,
    11, 10, 10, 11, 11, 11, 11, 11, 11, 10, 10, 11, 11, 10, 10, 11, 11, 11, 11, 11, 11, 11, 11, 10, 11, 11, 10, 10,
    10, 11, 11, 10, 10, 11, 11, 10, 10, 11, 11, 10, 9, 9, 10, 10, 10, 10, 10, 10, 9, 9, 9, 10, 10, 9, 10, 10, 9, 9,
    8, 9, 9, 9, 9, 9, 9, 9, 9, 8, 8, 9, 9, 8, 8, 7, 7, 8, 8, 7, 6, 6, 6, 6, 4, 4, 3, 1, 8, 8, 8, 8, 8, 8, 8, 8, 7,
    8, 8, 7, 7, 8, 8, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 8, 8, 9, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11,
    11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 11, 4, 11, 11, 11, 11, 12, 12, 11, 10, 11, 11, 10,
    10, 10, 10, 11, 11, 10, 10, 10, 10, 11, 11, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10,
    10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 11, 11, 10, 10, 10, 10,
    10, 10, 10, 10, 10, 10, 10, 10, 10, 11, 11, 10, 11, 11, 10, 9, 10, 10, 10, 10, 11, 11, 10, 9, 9, 10, 10, 9, 10,
    10, 10, 10, 9, 9, 10, 10, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9,
    9, 9, 9, 9, 9, 9, 9, 10, 10, 9, 9, 9, 10, 10, 8, 9, 9, 8, 8, 8, 8, 8, 8, 8, 8, 8, 8, 8, 8, 8, 9, 9, 8, 8, 8, 8,
    8, 8, 9, 9, 7, 8, 8, 7, 7, 7, 7, 7, 8, 8, 7, 7, 6, 6, 7, 7, 6, 5, 5, 6, 6, 4, 4, 4, 4};

__constant__ int32_t kSynthWindow[257] = {
    0, -1, -1, -1, -1, -1, -1, -2, -2, -2, -2, -3, -3, -4, -4, -5, -5, -6, -7, -7, -8, -9, -10, -11, -13, -14, -16,
    -17, -19, -21, -24, -26, -29, -31, -35, -38, -41, -45, -49, -53, -58, -63, -68, -73, -79, -85, -91, -97, -104,
    -111, -117, -125, -132, -139, -147, -154, -161, -169, -176, -183, -190, -196, -202, -208, 213, 218, 222, 225,
    227, 228, 228, 227, 224, 221, 215, 208, 200, 189, 177, 163, 146, 127, 106, 83, 57, 29, -2, -36, -72, -111, -153,
    -197, -244, -294, -347, -401, -459, -519, -581, -645, -711, -779, -848, -919, -991, -1064, -1137, -1210, -1283,
    -1356, -1428, -1498, -1567, -1634, -1698, -1759, -1817, -1870, -1919, -1962, -2001, -2032, -2057, -2075, -2085,
    -2087, -2080, -2063, 2037, 2000, 1952, 1893, 1822, 1739, 1644, 1535, 1414, 1280, 1131, 970, 794, 605, 402, 185,
    -45, -288, -545, -814, -1095, -1388, -1692, -2006, -2330, -2663, -3004, -3351, -3705, -4063, -4425, -4788,
    -5153, -5517, -5879, -6237, -6589, -6935, -7271, -7597, -7910, -8209, -8491, -8755, -8998, -9219, -9416, -9585,
    -9727, -9838, -9916, -9959, -9966, -9935, -9863, -9750, -9592, -9389, -9139, -8840, -8492, -8092, -7640, -7134,
    6574, 5959, 5288, 4561, 3776, 2935, 2037, 1082, 70, -998, -2122, -3300, -4533, -5818, -7154, -8540, -9975,
    -11455, -12980, -14548, -16155, -17799, -19478, -21189, -22929, -24694, -26482, -28289, -30112, -31947, -33791,
    -35640, -37489, -39336, -41176, -43006, -44821, -46617, -48390, -50137, -51853, -53534, -55178, -56778, -58333,
    -59838, -61289, -62684, -64019, -65290, -66494, -67629, -68692, -69679, -70590, -71420, -72169, -72835, -73415,
    -73908, -74313, -74630, -74856, -74992, 75038};

// scale-factor band widths by sampling_frequency index (44.1, 48, 32 kHz): 22 long bands, 13 short bands per window
__constant__ uint8_t cBandLong[3][22] = {
    {4, 4, 4, 4, 4, 4, 6, 6, 8, 8, 10, 12, 16, 20, 24, 28, 34, 42, 50, 54, 76, 158},
    {4, 4, 4, 4, 4, 4, 6, 6, 6, 8, 10, 12, 16, 18, 22, 28, 34, 40, 46, 54, 54, 192},
    {4, 4, 4, 4, 4, 4, 6, 6, 8, 10, 12, 16, 20, 24, 30, 38, 46, 56, 68, 84, 102, 26}};
__constant__ uint8_t cBandShort[3][13] = {{4, 4, 4, 4, 6, 8, 10, 12, 14, 18, 22, 30, 56},
                                          {4, 4, 4, 4, 6, 6, 10, 12, 14, 16, 20, 26, 66},
                                          {4, 4, 4, 4, 6, 8, 12, 16, 20, 26, 34, 42, 12}};
__constant__ uint8_t kPretab[22] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 3, 2, 0};
__constant__ uint8_t kSlen[16][2] = {{0, 0}, {0, 1}, {0, 2}, {0, 3}, {3, 0}, {1, 1}, {1, 2}, {1, 3},
                                     {2, 1}, {2, 2}, {2, 3}, {3, 1}, {3, 2}, {3, 3}, {4, 2}, {4, 3}};
// table_select -> code table (index into the 15 tables of kHuffLengths, -1: no bits) and linbits
__constant__ int8_t kTableOf[32] = {-1, 0, 1, 2, -1, 3, 4, 5, 6, 7, 8, 9, 10, 11, -1, 12,
                                    13, 13, 13, 13, 13, 13, 13, 13, 14, 14, 14, 14, 14, 14, 14, 14};
__constant__ uint8_t kLinbits[32] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                     1, 2, 3, 4, 6, 8, 10, 13, 4, 5, 6, 7, 8, 9, 11, 13};
__constant__ uint16_t kTableStart[16] = {0, 4, 13, 22, 38, 54, 90, 126, 162, 226, 290, 354, 610, 866, 1122, 1378};
// count1 table A by v << 3 | w << 2 | x << 1 | y
__constant__ uint8_t kQuadCodes[16] = {1, 5, 4, 5, 6, 5, 4, 4, 7, 3, 6, 0, 7, 2, 3, 1};
__constant__ uint8_t kQuadLengths[16] = {1, 4, 4, 5, 4, 6, 5, 6, 4, 5, 5, 6, 5, 6, 6, 6};
__constant__ float kCs[8] = {0.857492925712f, 0.881741997318f, 0.949628649103f, 0.983314592492f,
                             0.995517816065f, 0.999160558175f, 0.999899195243f, 0.999993155067f};
__constant__ float kCa[8] = {-0.514495755427f, -0.471731968565f, -0.313377454204f, -0.181913199611f,
                             -0.094574192526f, -0.040965582885f, -0.014198568572f, -0.003699974674f};

constexpr int kHuffEntries = 1378;
constexpr int kSfBytes = 64;       // per granule-channel: long [0, 22), short 22 + 3 * band + window
constexpr int kPow43 = 8207;       // |x|^(4/3) for |x| <= 8206
constexpr int kHybridThreads = 576;

// status codes; lib/mp3.py has the message of each
enum Mp3Status : int64_t {
  kZeroed = 1,          // main data begins before the first byte of the stream: the frame decodes as silence
  kReservedBlock = 2,   // window switching with block type 0
  kBigValues = 3,       // big_values above 288
  kMainData = 4,        // the part2_3 bits run past the main data available to the frame
  kGranuleEnd = 5,      // scale factors or big values run past the granule's part2_3_length
};

struct Granule {
  int64_t start;   // bit offset of the part2_3 data in the reservoir buffer
  int32_t p23, big, gain, sfc, ws, bt, mixed, ts[3], sbg[3], r0, r1, pre, sfs, c1, scfsi, skip;
};

}  // namespace

__global__ void __launch_bounds__(256) mp3_scan_kernel(const uint8_t* __restrict__ d, int64_t begin, int64_t end,
                                                       int64_t* __restrict__ cands, int max_cands,
                                                       int* __restrict__ count) {
  const int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool found = i + 4 <= end && d[i] == 0xFF && (d[i + 1] & 0xE0) == 0xE0;
  const int slot = warp_append(found, count, max_cands);
  if (slot < 0) return;
  cands[2 * (int64_t)slot] = i;
  cands[2 * (int64_t)slot + 1] = (int64_t)(((uint32_t)d[i] << 24) | ((uint32_t)d[i + 1] << 16) |
                                           ((uint32_t)d[i + 2] << 8) | d[i + 3]);
}

// one thread per frame: header and side info -> the frame's granule-channel descriptors and its status
__global__ void __launch_bounds__(128) mp3_side_info_kernel(const uint8_t* __restrict__ d, int64_t n_bytes,
                                                            const int64_t* __restrict__ frames,
                                                            const int64_t* __restrict__ md_off, int n_frames, int C,
                                                            Granule* __restrict__ gran, int64_t* __restrict__ fstatus) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  const int64_t off = frames[2 * f];
  const uint32_t h = (uint32_t)frames[2 * f + 1];
  const bool crc = ((h >> 16) & 1) == 0;
  PeekBits br{d, n_bytes, 8 * (off + 4 + (crc ? 2 : 0))};
  const int mdb = (int)br.read(9);
  br.read(C == 1 ? 5 : 3);
  const int scfsi0 = (int)br.read(4), scfsi1 = C == 2 ? (int)br.read(4) : 0;
  int64_t err = 0;
  const int64_t begin = md_off[f] - mdb;
  int64_t bit = 8 * begin;
  for (int gr = 0; gr < 2; ++gr) {
    for (int ch = 0; ch < C; ++ch) {
      Granule g;
      g.p23 = (int)br.read(12);
      g.big = (int)br.read(9);
      g.gain = (int)br.read(8);
      g.sfc = (int)br.read(4);
      g.ws = (int)br.read(1);
      if (g.ws) {
        g.bt = (int)br.read(2);
        g.mixed = (int)br.read(1);
        g.ts[0] = (int)br.read(5);
        g.ts[1] = (int)br.read(5);
        g.ts[2] = 0;
        g.sbg[0] = (int)br.read(3);
        g.sbg[1] = (int)br.read(3);
        g.sbg[2] = (int)br.read(3);
        g.r0 = g.r1 = 0;
        if (g.bt == 0 && !err) err = frame_status(kReservedBlock, br.pos - 8 * off - 3);
      } else {
        g.bt = g.mixed = 0;
        g.ts[0] = (int)br.read(5);
        g.ts[1] = (int)br.read(5);
        g.ts[2] = (int)br.read(5);
        g.sbg[0] = g.sbg[1] = g.sbg[2] = 0;
        g.r0 = (int)br.read(4);
        g.r1 = (int)br.read(3);
      }
      g.pre = (int)br.read(1);
      g.sfs = (int)br.read(1);
      g.c1 = (int)br.read(1);
      g.scfsi = gr == 1 ? (ch ? scfsi1 : scfsi0) : 0;
      if (g.big > 288 && !err) err = frame_status(kBigValues, 0);
      g.start = bit;
      bit += g.p23;
      g.skip = 0;
      gran[(int64_t)(2 * f + gr) * C + ch] = g;
    }
  }
  if (!err && begin < 0) err = frame_status(kZeroed, 0);
  if (!err && bit > 8 * md_off[f + 1]) err = frame_status(kMainData, bit - 8 * md_off[f + 1]);
  if (err) {
    for (int k = 0; k < 2 * C; ++k) gran[(int64_t)2 * f * C + k].skip = 1;
  }
  fstatus[f] = err;
}

// one CTA per frame: the frame's main data (after the header, CRC and side info) to its place in the reservoir buffer
__global__ void __launch_bounds__(128) mp3_gather_kernel(const uint8_t* __restrict__ d, const int64_t* __restrict__ frames,
                                                         const int64_t* __restrict__ md_off, int C,
                                                         uint8_t* __restrict__ md) {
  const int f = blockIdx.x;
  const uint32_t h = (uint32_t)frames[2 * f + 1];
  const int64_t src = frames[2 * f] + 4 + (((h >> 16) & 1) ? 0 : 2) + (C == 1 ? 17 : 32);
  const int64_t dst = md_off[f], len = md_off[f + 1] - md_off[f];
  for (int64_t k = threadIdx.x; k < len; k += blockDim.x) md[dst + k] = __ldg(d + src + k);
}

__global__ void mp3_pow43_kernel(float* __restrict__ pow43) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kPow43) pow43[i] = (float)pow((double)i, 4.0 / 3.0);
}

// one thread per granule-channel: scale factors, Huffman decoding and requantisation -> xr[576] (bitstream order)
__global__ void __launch_bounds__(128, 1) mp3_huffman_kernel(const uint8_t* __restrict__ md, int64_t md_bytes,
                                                          const Granule* __restrict__ gran, int n_gc, int C, int sr,
                                                          const float* __restrict__ pow43, float* __restrict__ xr,
                                                          uint8_t* __restrict__ sf_out, int64_t* __restrict__ gstatus) {
  __shared__ HuffBooks<uint8_t, kHuffEntries> bk;
  bk.build(kHuffSymbols, kHuffLengths, kTableStart, 15);
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_gc) return;
  const Granule g = gran[q];
  float* x = xr + (int64_t)q * 576;
  uint8_t* sf = sf_out + (int64_t)q * kSfBytes;
  for (int k = 0; k < kSfBytes; ++k) sf[k] = 0;
  int64_t err = 0;
  int k = 0;
  const bool shortb = g.ws && g.bt == 2;
  if (!g.skip) {
    PeekBits br{md, md_bytes, g.start, g.start + g.p23};
    const int s1 = kSlen[g.sfc][0], s2 = kSlen[g.sfc][1];
    if (shortb) {
      if (g.mixed)
        for (int b = 0; b < 8; ++b) sf[b] = (uint8_t)br.read(s1);
      for (int b = g.mixed ? 3 : 0; b < 12; ++b)
        for (int w = 0; w < 3; ++w) sf[22 + 3 * b + w] = (uint8_t)br.read(b < 6 ? s1 : s2);
    } else {
      // granule 1 re-reads granule 0's scale factors of the groups scfsi shares, from their known bit offset.  A short
      // granule 0 has long scale factors only in a mixed block's bands 0-7 (read at the start of its part2 data); the
      // other shared bands are 0 (oracle/mp3_oracle.py states the same rule).
      const Granule* g0 = g.scfsi ? &gran[q - C] : nullptr;
      const bool g0_short = g0 && g0->ws && g0->bt == 2, g0_mixed = g0_short && g0->mixed;
      int64_t p0 = g0 ? g0->start : 0;
      const int a0 = g0 ? kSlen[g0->sfc][0] : 0, b0 = g0 ? kSlen[g0->sfc][1] : 0;
#pragma unroll
      for (int grp = 0; grp < 4; ++grp) {
        const int first = grp == 0 ? 0 : 1 + 5 * grp, last = 6 + 5 * grp;   // bands 0-5, 6-10, 11-15, 16-20
        const int s = grp < 2 ? s1 : s2, s0 = grp < 2 ? a0 : b0;
        if (g.scfsi & (8 >> grp)) {
          if (g0_short) {
            for (int b = first; b < last; ++b) {
              PeekBits b0r{md, md_bytes, g0->start + (int64_t)b * a0};
              sf[b] = g0_mixed && b < 8 ? (uint8_t)b0r.read(a0) : 0;
            }
          } else {
            PeekBits b0r{md, md_bytes, p0};
            for (int b = first; b < last; ++b) sf[b] = (uint8_t)b0r.read(s0);
          }
        } else {
          for (int b = first; b < last; ++b) sf[b] = (uint8_t)br.read(s);
        }
        p0 += (int64_t)(last - first) * s0;
      }
    }
    if (br.over()) err = frame_status(kGranuleEnd, br.pos - g.start);
    // region boundaries in lines
    const int big = 2 * g.big;
    int r1, r2;
    if (g.ws) {
      r1 = 36;
      r2 = 576;
    } else {
      int a = 0, bnd1 = 0, bnd2 = 0;
      for (int b = 0; b < 22; ++b) {
        if (b == g.r0 + 1) bnd1 = a;
        if (b == min(g.r0 + g.r1 + 2, 22)) bnd2 = a;
        a += cBandLong[sr][b];
      }
      if (g.r0 + g.r1 + 2 >= 22) bnd2 = 576;
      r1 = bnd1;
      r2 = bnd2;
    }
    r1 = min(r1, big);
    r2 = min(r2, big);
    for (int reg = 0; reg < 3 && !err; ++reg) {
      const int stop = reg == 0 ? r1 : (reg == 1 ? r2 : big);
      const int ts = reg == 0 ? g.ts[0] : (reg == 1 ? g.ts[1] : g.ts[2]);
      const int t = kTableOf[ts];
      if (t < 0) {
        for (; k < stop; ++k) x[k] = 0.0f;
        continue;
      }
      const int lb = kLinbits[ts];
      const int first = kTableStart[t], last = kTableStart[t + 1];
      for (; k < stop; k += 2) {
        const int sym = bk.sym[bk.decode(br, first, last)];
        int vx = sym >> 4, vy = sym & 15;
        if (lb && vx == 15) vx += (int)br.read(lb);
        if (vx && br.read(1)) vx = -vx;
        if (lb && vy == 15) vy += (int)br.read(lb);
        if (vy && br.read(1)) vy = -vy;
        x[k] = (float)vx;
        x[k + 1] = (float)vy;
      }
      if (br.over()) err = frame_status(kGranuleEnd, br.pos - g.start);
    }
    while (!err && k <= 572 && br.pos < br.end) {
      int v;
      if (g.c1) {
        v = 15 - (int)br.read(4);
      } else {
        const uint32_t w = br.peek32();
        v = -1;
        for (int c = 0; c < 16 && v < 0; ++c)
          if ((w >> (32 - kQuadLengths[c])) == kQuadCodes[c]) v = c;
        br.pos += kQuadLengths[v];
      }
      float qv[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int bit = (v >> (3 - j)) & 1;
        qv[j] = bit ? (br.read(1) ? -1.0f : 1.0f) : 0.0f;
      }
      if (br.over()) break;   // a quadruple that crosses the granule's end is dropped
#pragma unroll
      for (int j = 0; j < 4; ++j) x[k + j] = qv[j];
      k += 4;
    }
  }
  if (err || g.skip) k = 0;
  for (int j = k; j < 576; ++j) x[j] = 0.0f;
  gstatus[q] = err;
  if (err || g.skip || k == 0) return;
  // requantisation in place, band by band
  const int m = g.sfs ? 4 : 2;   // quarter steps per scale-factor step
  int j = 0;
  if (!shortb || g.mixed) {
    const int nb = shortb ? 8 : 22;
    for (int b = 0; b < nb && j < k; ++b) {
      const float s = exp2_quarter(g.gain - 210 - m * (sf[b] + (g.pre ? kPretab[b] : 0)));
      for (int e = j + cBandLong[sr][b]; j < e; ++j) {
        const float v = x[j];
        const int a = (int)fabsf(v);
        x[j] = copysignf(pow43[min(a, kPow43 - 1)] * s, v);
      }
    }
  }
  if (shortb) {
    for (int b = g.mixed ? 3 : 0; b < 13 && j < k; ++b) {
      const int n = cBandShort[sr][b];
#pragma unroll
      for (int w = 0; w < 3; ++w) {
        const float s = exp2_quarter(g.gain - 210 - 8 * g.sbg[w] - m * sf[22 + 3 * b + w]);
        for (int e = j + n; j < e; ++j) {
          const float v = x[j];
          const int a = (int)fabsf(v);
          x[j] = copysignf(pow43[min(a, kPow43 - 1)] * s, v);
        }
      }
    }
  }
}

__device__ __forceinline__ void ms_band(float* __restrict__ l, float* __restrict__ r, int n) {
  const float s = 0.70710678118654752f;
  for (int j = 0; j < n; ++j) {
    const float a = l[j], b = r[j];
    l[j] = (a + b) * s;
    r[j] = (a - b) * s;
  }
}

__device__ __forceinline__ bool band_nonzero(const float* __restrict__ r, int n) {
  for (int j = 0; j < n; ++j)
    if (r[j] != 0.0f) return true;
  return false;
}

// MPEG-1 intensity gains of is_pos 0..6: left tan(p pi / 12) / (1 + tan(p pi / 12)), right 1 / (1 + tan(p pi / 12))
__constant__ float kIsLeft[7] = {0.0f, 2.113248654052e-01f, 3.660254037844e-01f, 5.0e-01f, 6.339745962156e-01f,
                                 7.886751345948e-01f, 1.0f};

__device__ __forceinline__ void is_band(float* __restrict__ l, float* __restrict__ r, int n, int pos) {
  const float gl = kIsLeft[pos], gr = kIsLeft[6 - pos];
  for (int j = 0; j < n; ++j) {
    const float a = l[j];
    l[j] = a * gl;
    r[j] = a * gr;
  }
}

// one thread per joint-stereo granule: MS and MPEG-1 intensity stereo in place (bitstream order)
__global__ void __launch_bounds__(128) mp3_stereo_kernel(const int64_t* __restrict__ frames,
                                                         const Granule* __restrict__ gran,
                                                         const uint8_t* __restrict__ sf_all, int n_granules, int sr,
                                                         float* __restrict__ xr) {
  const int gi = blockIdx.x * blockDim.x + threadIdx.x;
  if (gi >= n_granules) return;
  const uint32_t h = (uint32_t)frames[2 * (gi >> 1) + 1];
  if (((h >> 6) & 3) != 1) return;
  const int modex = (h >> 4) & 3;
  const Granule& g1 = gran[2 * gi + 1];
  if (g1.skip || gran[2 * gi].skip || !modex) return;
  float* l = xr + (int64_t)(2 * gi) * 576;
  float* r = l + 576;
  const bool ms = modex & 2;
  if (!(modex & 1)) {
    ms_band(l, r, 576);
    return;
  }
  const uint8_t* sf = sf_all + (int64_t)(2 * gi + 1) * kSfBytes;
  const bool shortb = g1.ws && g1.bt == 2;
  const int long_end = shortb ? (g1.mixed ? 8 : 0) : 22;
  int p = 576;
  bool nz = false;
  if (shortb) {
    int found = 0;   // bit w: window w has a nonzero band at or above this one
    for (int b = 12; b >= (g1.mixed ? 3 : 0); --b) {
      const int n = cBandShort[sr][b];
      for (int w = 2; w >= 0; --w) {
        p -= n;
        if (!(found >> w & 1) && band_nonzero(r + p, n)) found |= 1 << w;
        const int pos = sf[22 + 3 * (b == 12 ? 11 : b) + w];
        if ((found >> w & 1) || pos >= 7) {
          if (ms) ms_band(l + p, r + p, n);
        } else {
          is_band(l + p, r + p, n, pos);
        }
      }
    }
    nz = found != 0;
  }
  for (int b = long_end - 1; b >= 0; --b) {
    const int n = cBandLong[sr][b];
    p -= n;
    if (!nz && band_nonzero(r + p, n)) nz = true;
    const int pos = sf[b == 21 ? 20 : b];
    if (nz || pos >= 7) {
      if (ms) ms_band(l + p, r + p, n);
    } else {
      is_band(l + p, r + p, n, pos);
    }
  }
}

// xr (bitstream order) of granule-channel q, reordered to (subband, 3 * k + window) for short blocks, into s[576]
__device__ __forceinline__ void load_reordered(const float* __restrict__ x, const Granule& g, int sr, float* s) {
  for (int j = threadIdx.x; j < 576; j += blockDim.x) {
    int dst = j;
    if (g.ws && g.bt == 2 && !(g.mixed && j < 36)) {
      int p0 = g.mixed ? 36 : 0;
      for (int b = g.mixed ? 3 : 0; b < 13; ++b) {
        const int n = cBandShort[sr][b];
        if (j < p0 + 3 * n) {
          const int r = j - p0;
          dst = p0 + 3 * (r % n) + r / n;
          break;
        }
        p0 += 3 * n;
      }
    }
    s[dst] = x[j];
  }
}

__device__ __forceinline__ void antialias(float* s, const Granule& g) {
  const bool shortb = g.ws && g.bt == 2;
  const int nb = shortb ? (g.mixed ? 1 : 0) : 31;
  for (int t = threadIdx.x; t < nb * 8; t += blockDim.x) {
    const int sb = t >> 3, i = t & 7;
    const float a = s[18 * sb + 17 - i], b = s[18 * (sb + 1) + i];
    s[18 * sb + 17 - i] = a * kCs[i] - b * kCa[i];
    s[18 * (sb + 1) + i] = b * kCs[i] + a * kCa[i];
  }
}

// output i (0..35) of subband sb's windowed IMDCT; cos144[m] = cos(pi m / 72)
__device__ __forceinline__ float imdct_at(const float* s, const Granule& g, int sb, int i, const float* cos144,
                                          const float (*win)[36]) {
  const bool shortb = g.ws && g.bt == 2 && !(g.mixed && sb < 2);
  const float* x = s + 18 * sb;
  if (!shortb) {
    float acc = 0.0f;
    const int bt = (g.ws && g.bt == 2) ? 0 : g.bt;
#pragma unroll
    for (int k = 0; k < 18; ++k) acc += x[k] * cos144[((2 * i + 19) * (2 * k + 1)) % 144];
    return acc * win[bt][i];
  }
  float acc = 0.0f;
#pragma unroll
  for (int w = 0; w < 3; ++w) {
    const int ii = i - 6 - 6 * w;
    if (ii < 0 || ii >= 12) continue;
    float a = 0.0f;
#pragma unroll
    for (int k = 0; k < 6; ++k) a += x[3 * k + w] * cos144[(3 * (2 * ii + 7) * (2 * k + 1)) % 144];
    acc += a * win[2][ii];
  }
  return acc;
}

// one CTA per granule-channel: reorder, antialias, IMDCT with overlap of the previous granule's tail (recomputed from
// its spectrum), frequency inversion, then the 64-value V vector of each of the 18 subband slots
__global__ void __launch_bounds__(kHybridThreads) mp3_hybrid_kernel(const Granule* __restrict__ gran,
                                                                    const float* __restrict__ xr, int n_granules, int C,
                                                                    int sr, float* __restrict__ V) {
  __shared__ float cur[576], prev[576], S[18][32];
  __shared__ float cos144[144], cos128[128], win[4][36];
  const int q = blockIdx.x, gi = q / C, ch = q % C;
  const int t = threadIdx.x;
  if (t < 144) cos144[t] = (float)cospi(t / 72.0);
  if (t < 128) cos128[t] = (float)cospi(t / 64.0);
  if (t < 36) {
    const double l = sinpi((t + 0.5) / 36.0);
    win[0][t] = (float)l;
    win[1][t] = (float)(t < 18 ? l : t < 24 ? 1.0 : t < 30 ? sinpi((t - 18 + 0.5) / 12.0) : 0.0);
    win[3][t] = (float)(t < 6 ? 0.0 : t < 12 ? sinpi((t - 6 + 0.5) / 12.0) : t < 18 ? 1.0 : l);
    win[2][t] = t < 12 ? (float)sinpi((t + 0.5) / 12.0) : 0.0f;
  }
  const Granule g = gran[q];
  load_reordered(xr + (int64_t)q * 576, g, sr, cur);
  Granule gp = g;
  if (gi > 0) {
    gp = gran[q - C];
    load_reordered(xr + (int64_t)(q - C) * 576, gp, sr, prev);
  } else {
    for (int j = t; j < 576; j += blockDim.x) prev[j] = 0.0f;
  }
  __syncthreads();
  antialias(cur, g);
  if (gi > 0) antialias(prev, gp);
  __syncthreads();
  {
    const int sb = t / 18, i = t % 18;
    float v = imdct_at(cur, g, sb, i, cos144, win) + imdct_at(prev, gp, sb, 18 + i, cos144, win);
    if ((sb & 1) && (i & 1)) v = -v;
    S[i][sb] = v;
  }
  __syncthreads();
  float* out = V + ((int64_t)ch * n_granules * 18 + (int64_t)gi * 18) * 64;
  for (int o = t; o < 18 * 64; o += blockDim.x) {
    const int slot = o >> 6, i = o & 63;
    float acc = 0.0f;
#pragma unroll 8
    for (int k = 0; k < 32; ++k) acc += S[slot][k] * cos128[((16 + i) * (2 * k + 1)) & 127];
    out[o] = acc;
  }
}

// one thread per output sample: the window D over the 16 V vectors up to the sample's slot (zero before the stream)
__global__ void __launch_bounds__(256) mp3_window_kernel(const float* __restrict__ V, int64_t slots, int C,
                                                         float* __restrict__ out) {
  __shared__ float D[512];
  for (int i = threadIdx.x; i < 257; i += blockDim.x) {
    const float v = (float)kSynthWindow[i] * (1.0f / 65536.0f);
    D[i] = v;
    if (i) D[512 - i] = (i & 63) ? -v : v;
  }
  __syncthreads();
  const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= slots * 32 * C) return;
  const int ch = (int)(o / (slots * 32));
  const int64_t r = o - (int64_t)ch * slots * 32;
  const int64_t t = r >> 5;
  const int j = (int)(r & 31);
  const float* v = V + (int64_t)ch * slots * 64;
  float acc = 0.0f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t a = t - 2 * i, b = t - 2 * i - 1;
    if (a >= 0) acc += v[a * 64 + j] * D[64 * i + j];
    if (b >= 0) acc += v[b * 64 + 32 + j] * D[64 * i + 32 + j];
  }
  out[(int64_t)ch * slots * 32 + t * 32 + j] = acc;
}

// status[f]: the frame's own status, else the first of its granule-channels'
__global__ void mp3_status_kernel(const int64_t* __restrict__ fstatus, const int64_t* __restrict__ gstatus,
                                  int n_frames, int C, int64_t* __restrict__ status) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  int64_t s = fstatus[f];
  for (int k = 0; k < 2 * C && !s; ++k) s = gstatus[(int64_t)2 * f * C + k];
  status[f] = s;
}

namespace {

struct Mp3Workspace {
  uint8_t* md;
  Granule* gran;
  int64_t* fstatus;
  int64_t* gstatus;
  uint8_t* sf;
  float* xr;
  float* V;
  float* pow43;
  int64_t bytes;
};

Mp3Workspace carve(uint8_t* base, int64_t n_frames, int C, int64_t md_bytes) {
  Mp3Workspace w{};
  Carver c{base};
  const int64_t gc = 2 * n_frames * C;
  w.md = c.take(md_bytes + 8);
  w.gran = c.take<Granule>(gc * (int64_t)sizeof(Granule));
  w.fstatus = c.take<int64_t>(n_frames * 8);
  w.gstatus = c.take<int64_t>(gc * 8);
  w.sf = c.take(gc * kSfBytes);
  w.xr = c.take<float>(gc * 576 * 4);
  w.V = c.take<float>((int64_t)C * n_frames * 36 * 64 * 4);
  w.pow43 = c.take<float>(kPow43 * 4);
  w.bytes = c.bytes;
  return w;
}

}  // namespace

int64_t mp3_workspace_bytes(int64_t n_frames, int channels, int64_t md_bytes) {
  if (n_frames < 0 || channels < 1 || channels > 2 || md_bytes < 0) return -1;
  return carve(nullptr, n_frames, channels, md_bytes).bytes;
}

cudaError_t launch_mp3_scan(const uint8_t* data, int64_t begin, int64_t end, int64_t* cands, int max_cands, int* count,
                            cudaStream_t stream) {
  if (!data || !cands || !count || begin < 0 || end < begin || max_cands < 0) return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(count, 0, sizeof(int), stream);
  if (e != cudaSuccess || end == begin) return e;
  const int64_t threads = end - begin;
  mp3_scan_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(data, begin, end, cands, max_cands, count);
  return cudaGetLastError();
}

cudaError_t launch_mp3_decode(const uint8_t* data, int64_t n_bytes, const int64_t* frames, const int64_t* md_off,
                              int n_frames, int channels, int rate_index, int64_t md_bytes, void* workspace,
                              int64_t workspace_bytes, float* out, int64_t* status, cudaStream_t stream) {
  if (!data || !frames || !md_off || !workspace || !out || !status || n_frames < 1 || channels < 1 || channels > 2 ||
      rate_index < 0 || rate_index > 2 || md_bytes < 0 || workspace_bytes < mp3_workspace_bytes(n_frames, channels,
                                                                                              md_bytes))
    return cudaErrorInvalidValue;
  Mp3Workspace w = carve(static_cast<uint8_t*>(workspace), n_frames, channels, md_bytes);
  const int C = channels, G = 2 * n_frames, gc = G * C;
  mp3_pow43_kernel<<<(kPow43 + 255) / 256, 256, 0, stream>>>(w.pow43);
  mp3_side_info_kernel<<<(n_frames + 127) / 128, 128, 0, stream>>>(data, n_bytes, frames, md_off, n_frames, C, w.gran,
                                                                   w.fstatus);
  mp3_gather_kernel<<<n_frames, 128, 0, stream>>>(data, frames, md_off, C, w.md);
  mp3_huffman_kernel<<<(gc + 127) / 128, 128, 0, stream>>>(w.md, md_bytes, w.gran, gc, C, rate_index, w.pow43, w.xr,
                                                           w.sf, w.gstatus);
  if (C == 2) mp3_stereo_kernel<<<(G + 127) / 128, 128, 0, stream>>>(frames, w.gran, w.sf, G, rate_index, w.xr);
  mp3_hybrid_kernel<<<gc, kHybridThreads, 0, stream>>>(w.gran, w.xr, G, C, rate_index, w.V);
  const int64_t slots = (int64_t)G * 18;
  const int64_t n_out = slots * 32 * C;
  mp3_window_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, stream>>>(w.V, slots, C, out);
  mp3_status_kernel<<<(n_frames + 127) / 128, 128, 0, stream>>>(w.fstatus, w.gstatus, n_frames, C, status);
  return cudaGetLastError();
}

}  // namespace vr
