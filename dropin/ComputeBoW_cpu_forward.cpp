// Compiled with the SAME rename as the reference's src/Frame.cpp and src/KeyFrame.cpp (COMPILE_DEFINITIONS "ComputeBoW=ComputeBoW_cpu"), so inside
// this file ComputeBoW names the reference's own CPU bodies. It exports them as free functions for A/B runs and for the link-and-run test
// (tests/test_gpu_compute_bow.py), which transforms the same objects with both implementations.
#include "Frame.h"
#include "KeyFrame.h"

void cslam_cpu_Frame_ComputeBoW(Frame& F) { F.ComputeBoW(); }
void cslam_cpu_KeyFrame_ComputeBoW(KeyFrame* pKF) { pKF->ComputeBoW(); }
