#!/usr/bin/env python
"""Twin of the reference's evaluation sample (modules/optflow/samples/optical_flow_evaluation.cpp):

    python tools/flow_eval.py image1 image2 {tvl1,farneback,brox,denselk,dis_ultrafast,dis_fast,dis_medium,fastbm}
                              [groundtruth.flo]
                              [-m endpoint|angular|angular-fixed] [-o out.flo]

computes the flow between two images on the GPU, optionally writes it as a Middlebury .flo file and, given a
ground truth, prints the sample's statistics (average, standard deviation, R0.5..R10, A0.50..A0.95).
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("image1")
    ap.add_argument("image2")
    ap.add_argument("algorithm", choices=["tvl1", "farneback", "brox", "denselk", "dis_ultrafast", "dis_fast",
                                                  "dis_medium", "fastbm"])
    ap.add_argument("groundtruth", nargs="?")
    ap.add_argument("-m", "--measure", default="endpoint", choices=["endpoint", "angular", "angular-fixed"])
    ap.add_argument("-o", "--out")
    a = ap.parse_args()
    import cv2
    import numpy as np
    import torch
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200 import flowio
    i1, i2 = cv2.imread(a.image1, cv2.IMREAD_GRAYSCALE), cv2.imread(a.image2, cv2.IMREAD_GRAYSCALE)
    if i1 is None or i2 is None or i1.shape != i2.shape:
        sys.exit("cannot read the images, or their sizes differ")
    dev = torch.device("cuda:0")
    if a.algorithm == "brox":
        alg = ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, 10, 77, 10)
        d1, d2 = (torch.from_numpy((x / np.float32(255)).astype(np.float32)).to(dev) for x in (i1, i2))
    elif a.algorithm.startswith("dis_"):
        alg = ocb.DISOpticalFlow_create({"dis_ultrafast": ocb.DISOPTICAL_FLOW_PRESET_ULTRAFAST,
                                         "dis_fast": ocb.DISOPTICAL_FLOW_PRESET_FAST,
                                         "dis_medium": ocb.DISOPTICAL_FLOW_PRESET_MEDIUM}[a.algorithm])
        d1, d2 = torch.from_numpy(i1).to(dev), torch.from_numpy(i2).to(dev)
    else:
        alg = {"tvl1": ocb.OpticalFlowDual_TVL1_create, "farneback": ocb.FarnebackOpticalFlow_create,
               "denselk": ocb.DensePyrLKOpticalFlow_create, "fastbm": ocb.FastOpticalFlowBM}[a.algorithm]()
        d1, d2 = torch.from_numpy(i1).to(dev), torch.from_numpy(i2).to(dev)
    flow = alg.calc(d1, d2, torch.zeros((*i1.shape, 2), dtype=torch.float32, device=dev))
    torch.cuda.synchronize()
    flow = flow.cpu().numpy()
    if a.out:
        flowio.writeOpticalFlow(a.out, flow)
    if a.groundtruth:
        gt = flowio.readOpticalFlow(a.groundtruth)
        if gt.shape != flow.shape:
            sys.exit("ground truth size differs from the images")
        measure = {"endpoint": flowio.ERR_ENDPOINT, "angular": flowio.ERR_ANGULAR_REFERENCE,
                   "angular-fixed": flowio.ERR_ANGULAR}[a.measure]
        st = flowio.errorStats(flowio.errorMap(flow, gt, measure))
        print("Average: %.2f\nStandard deviation: %.2f" % (st["mean"], st["std"]))
        for k, v in st["R"].items():
            print("R%.1f: %.2f%%" % (k, v * 100))
        for k, v in st["A"].items():
            print("A%.2f: %.2f" % (k, v))
        print("accuracy (EPE <= 0.1 px): %.4f" % flowio.accuracy(gt, flow, 0.1))


if __name__ == "__main__":
    main()
