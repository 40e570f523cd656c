#!/usr/bin/env python
"""N single IcpFast alignments of the benchmark pair (one in flight, default options, host buffers):
the launch sequence of bench.py's roofline measurement.  argv[2] = knn_queries_per_cta (0: one query
per thread = icp_knn_kernel; 1024: the launch shape bench.py uses with many alignments in flight =
icp_knn_batch_kernel)."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
import staticmapping_b200 as smb
n = int(sys.argv[1]) if len(sys.argv) > 1 else 3
src, sub, _ = bench.make_workload(0)
tgt = smb.CalculateNormals(sub)
m = smb.IcpFast(0)
qpc = int(sys.argv[2]) if len(sys.argv) > 2 else 0
m.InitWithXml({"max_iteration": 30, "disable_convergence_check": 1, "use_graphs": 0, "knn_queries_per_cta": qpc})
for _ in range(n):
    m.SetInputSource(smb.EigenCloud(src)); m.SetInputTarget(smb.EigenCloud(tgt.points, tgt.normals))
    ok, res = m.Align(np.eye(4))
print("iterations", m.GetAlignInfo()["iterations"], "score", m.GetFitnessScore())
