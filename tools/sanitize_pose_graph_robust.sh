# compute-sanitizer memcheck over one small robust pose-graph run: 300 nodes of the seq-05-shaped graph of
# tests/test_pose_graph.py with a loop edge at every 40th node and two false loops, so that the weighted stages, the
# residual and weight kernels and the weights download all run.
#   bash tools/sanitize_pose_graph_robust.sh   (from the repository root, on a GPU machine with compute-sanitizer)
cat > /tmp/pgr_small.py <<PY
import sys; sys.path.insert(0, "."); sys.path.insert(0, "tests")
import numpy as np
import pose_graph_oracle as pgo
from test_pose_graph import device_graph, seq_graph
G, O, _ = seq_graph("05")
O, G = O[:300], G[:300]
loops = [(k - 40, k, pgo.inv_mul(G[k - 40], G[k])) for k in range(40, 300, 40)]
loops += [(10, 200, np.eye(4)), (50, 250, pgo.inv_mul(G[50], G[250]) @ pgo.exp4([5.0, 0, 0, 0, 0, 0.3]))]
r = device_graph(O, loops)
print("robust", r.pose_graph_optimize_robust())
print("weights", r.pose_graph_loop_weights())
r.close()
PY
echo "== memcheck: robust pose graph"
timeout 900 compute-sanitizer --tool memcheck --print-limit 5 python /tmp/pgr_small.py 2>&1 | tail -6
