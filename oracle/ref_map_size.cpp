// ORACLE - TEST INFRASTRUCTURE ONLY.  Our own translation unit, linked by oracle/build_ref.py into a second build of the
// unmodified reference association extension (dapalib_ref_dims).  The reference hard-codes the heat-map size in one
// global with external linkage (`vector<int> heatmapDim = {43, 128, 208}`, association.cpp); extract() allocates, copies
// and launches from it, and connect() indexes the depth map by its own shape.  Setting that global from here runs the
// same reference code at other map sizes without changing a line of it.
//
// The reference's NMS is deterministic only at some sizes, and the setter refuses every other one:
//   * w % 16 != 0: nmsRegisterKernel rounds its grid up to 16 x 16 blocks; threads with x >= w on row 0 take the border
//     branch and write 0 to index x, which is row 1, column x - w, racing with the real flag of that pixel;
//   * h * w % 512 != 0: writeResultKernel has a __syncthreads() inside `if (globalIdx < length)`, which a partial last
//     block would reach divergently (undefined behaviour).
// (h % 16 != 0 is harmless: the extra rows only write 0 at columns 0 and w - 1, border pixels of the next plane.)
#include <vector>

extern std::vector<int> heatmapDim;

extern "C" __attribute__((visibility("default"))) int ref_map_size_check(int h, int w) {
    if (h < 3 || w < 3) return 1;         // no interior pixel
    if (w % 16 != 0) return 2;            // racing border writes of nmsRegisterKernel
    if ((h * w) % 512 != 0) return 3;     // divergent __syncthreads() in writeResultKernel
    return 0;
}

// Sets the map size the reference module runs at: 0, or the refusal code of ref_map_size_check (nothing is changed).
extern "C" __attribute__((visibility("default"))) int ref_set_map_size(int h, int w) {
    const int rc = ref_map_size_check(h, w);
    if (rc != 0) return rc;
    heatmapDim = {43, h, w};
    return 0;
}

// The size the reference module currently runs at (h, w).
extern "C" __attribute__((visibility("default"))) void ref_get_map_size(int* h, int* w) {
    *h = heatmapDim[1];
    *w = heatmapDim[2];
}
