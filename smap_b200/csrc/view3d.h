// The 3D panel of smapb_encode_jpeg_ex(SMAPB_ENCODE_VIEW3D) (view3d.cu): the skeletons of a record's pred3d, seen from
// lib/visualize/vis.py's viewpoint, painted as labels into the panel's columns of the encoder's label plane.
#pragma once
#include <cuda_runtime.h>

#include "../../include/smap_b200.h"

namespace smapb {

// Panel elements: the 12 edges of the fit box, then limb k of row p at PANEL_BOX + p * SMAPB_NL + k.
constexpr int PANEL_BOX = 12;
constexpr int PANEL_ELEMS = PANEL_BOX + SMAPB_MAXP * SMAPB_NL;
// A panel label is (paint order + 1) << 3 | colour: the colour is the palette index p % 6 of a limb's person, or
// PANEL_GREY for a box edge; 0 is the white background.  atomicMax keeps the last element in paint order.
constexpr int PANEL_GREY = 6;

struct PanelImg {
    const smapb_record* rec;
    int P;  // the panel is P x P (P = the frame's height)
    int stride;  // row length of the label plane
    long long base;  // label of the panel's pixel (0, 0)
};

// one element: its end points in panel pixels and its label (0: not drawn)
struct PanelSeg {
    int ax, ay, bx, by, label;
};

// Launches the set-up (one CTA per image) and the paint (one CTA per element) for n panels: imgs device [n], segs device
// [n][PANEL_ELEMS] scratch, labels the zeroed label plane the imgs point into.  The caller checks cudaGetLastError.
void panel_launch(const PanelImg* imgs, int n, PanelSeg* segs, int* labels, cudaStream_t st);

}  // namespace smapb
