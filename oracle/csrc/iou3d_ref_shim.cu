// TEST INFRASTRUCTURE (see oracle/__init__.py).  C-linkage doors onto the REFERENCE's own rotated-box IoU / NMS launchers
// (pcdet/ops/iou3d_nms/src/iou3d_nms_kernel.cu:378-414), which oracle/iou3d_ref_build.py compiles from the source where it
// lies (never copied) into oracle/_ref/libiou3d_nms_ref.so.  The launchers use the legacy default stream.
//
// ref_nms restates the host side of the reference's nms_gpu / nms_normal_gpu (iou3d_nms.cpp:90-186) around the launcher:
// cudaMalloc of the full N x ceil(N/64) mask, the mask kernel, a blocking cudaMemcpy to the host, cudaFree, and the greedy
// pass on the CPU.  Returns the kept count (keep: host int64[N]) or -1 on a CUDA error.
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

void boxesoverlapLauncher(const int num_a, const float* boxes_a, const int num_b, const float* boxes_b, float* ans_overlap);
void boxesioubevLauncher(const int num_a, const float* boxes_a, const int num_b, const float* boxes_b, float* ans_iou);
void nmsLauncher(const float* boxes, unsigned long long* mask, int boxes_num, float nms_overlap_thresh);
void nmsNormalLauncher(const float* boxes, unsigned long long* mask, int boxes_num, float nms_overlap_thresh);

extern "C" void ref_boxes_overlap_bev(int num_a, const float* boxes_a, int num_b, const float* boxes_b, float* out) {
    boxesoverlapLauncher(num_a, boxes_a, num_b, boxes_b, out);
}

extern "C" void ref_boxes_iou_bev(int num_a, const float* boxes_a, int num_b, const float* boxes_b, float* out) {
    boxesioubevLauncher(num_a, boxes_a, num_b, boxes_b, out);
}

extern "C" int ref_nms(const float* boxes, int boxes_num, float thresh, int normal, int64_t* keep) {
    if (boxes_num <= 0) return 0;
    const int col_blocks = (boxes_num + 63) / 64;
    unsigned long long* mask = nullptr;
    if (cudaMalloc((void**)&mask, (size_t)boxes_num * col_blocks * sizeof(unsigned long long)) != cudaSuccess) return -1;
    if (normal) nmsNormalLauncher(boxes, mask, boxes_num, thresh);
    else nmsLauncher(boxes, mask, boxes_num, thresh);
    std::vector<unsigned long long> mask_cpu((size_t)boxes_num * col_blocks);
    const cudaError_t e = cudaMemcpy(mask_cpu.data(), mask, mask_cpu.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
    cudaFree(mask);
    if (e != cudaSuccess) return -1;
    std::vector<unsigned long long> remv(col_blocks, 0);
    int num_to_keep = 0;
    for (int i = 0; i < boxes_num; i++) {
        const int nblock = i / 64, inblock = i % 64;
        if (!(remv[nblock] & (1ULL << inblock))) {
            keep[num_to_keep++] = i;
            const unsigned long long* p = mask_cpu.data() + (size_t)i * col_blocks;
            for (int j = nblock; j < col_blocks; j++) remv[j] |= p[j];
        }
    }
    return num_to_keep;
}
