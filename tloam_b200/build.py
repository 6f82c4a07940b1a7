"""In-tree build of libtloam_b200.so, libtloam_b200_gmi.so, libtloam_b200_unpack.so, libtloam_b200_deskew.so,
libtloam_b200_loop.so, libtloam_b200_loopv.so, libtloam_b200_pg.so, libtloam_b200_gmc.so, libtloam_b200_pgr.so,
libtloam_b200_loopvs.so, libtloam_b200_gmd.so, libtloam_b200_gmm.so, libtloam_b200_loc.so, libtloam_b200_reloc.so,
libtloam_b200_mapu.so, libtloam_b200_occ.so, libtloam_b200_dist.so, libtloam_b200_plan.so, libtloam_b200_greg.so,
libtloam_b200_frontier.so and libtloam_b200_terrain.so (hand-written CUDA for sm_90a; no torch, no CPU fallback).

    python -m tloam_b200.build [--force]

nvcc cross-compiles without a GPU; the .so files are git-ignored and built in the tree.  libtloam_b200_gmi.so holds the
global map's intensity kernels (csrc/gmap_intensity.cu), libtloam_b200_unpack.so the packed-scan unpacking kernel
(csrc/unpack_scan.cu), libtloam_b200_deskew.so the motion-correction kernels (csrc/deskew.cu), libtloam_b200_loop.so the
loop-closure kernels (csrc/scan_context.cu), libtloam_b200_loopv.so the loop-verification kernels (csrc/loop_verify.cu),
libtloam_b200_pg.so the pose-graph kernels (csrc/pose_graph.cu), libtloam_b200_gmc.so the global map's pose tables and
loop-closure correction (csrc/map_correct.cu), libtloam_b200_pgr.so the robust pose graph's loop-edge weights
(csrc/pose_graph_robust.cu), libtloam_b200_loopvs.so the loop verification against a submap (csrc/loop_verify_submap.cu), libtloam_b200_gmd.so the
global map's dynamic-point removal (csrc/map_dynamic.cu), libtloam_b200_gmm.so the merge of the global map into one voxel
grid (csrc/map_merge.cu), libtloam_b200_loc.so the localization in a prior map (csrc/localize.cu), libtloam_b200_reloc.so the relocalization in a
prior map (csrc/relocalize.cu), libtloam_b200_mapu.so the update of a prior map (csrc/map_update.cu), libtloam_b200_occ.so the occupancy grid of the global
map (csrc/occupancy.cu), libtloam_b200_dist.so the distance field and costmap of an occupancy grid (csrc/distance.cu),
libtloam_b200_plan.so the path planning on that costmap (csrc/plan.cu), libtloam_b200_greg.so the global registration
of two clouds (csrc/global_registration.cu), libtloam_b200_frontier.so the exploration frontiers of the costmap
(csrc/frontier.cu), libtloam_b200_terrain.so the terrain map of a cloud (csrc/terrain.cu); libtloam_b200.so loads each from its own directory when first needed.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libtloam_b200.so")
SOURCES = [os.path.join(CSRC, "tloam_b200.cu")]
GMI_LIB = os.path.join(HERE, "libtloam_b200_gmi.so")
GMI_SOURCES = [os.path.join(CSRC, "gmap_intensity.cu")]
UNPACK_LIB = os.path.join(HERE, "libtloam_b200_unpack.so")
UNPACK_SOURCES = [os.path.join(CSRC, "unpack_scan.cu")]
DESKEW_LIB = os.path.join(HERE, "libtloam_b200_deskew.so")
DESKEW_SOURCES = [os.path.join(CSRC, "deskew.cu")]
LOOP_LIB = os.path.join(HERE, "libtloam_b200_loop.so")
LOOP_SOURCES = [os.path.join(CSRC, "scan_context.cu")]
LOOPV_LIB = os.path.join(HERE, "libtloam_b200_loopv.so")
LOOPV_SOURCES = [os.path.join(CSRC, "loop_verify.cu")]
PG_LIB = os.path.join(HERE, "libtloam_b200_pg.so")
PG_SOURCES = [os.path.join(CSRC, "pose_graph.cu")]
GMC_LIB = os.path.join(HERE, "libtloam_b200_gmc.so")
GMC_SOURCES = [os.path.join(CSRC, "map_correct.cu")]
PGR_LIB = os.path.join(HERE, "libtloam_b200_pgr.so")
PGR_SOURCES = [os.path.join(CSRC, "pose_graph_robust.cu")]
LOOPVS_LIB = os.path.join(HERE, "libtloam_b200_loopvs.so")
LOOPVS_SOURCES = [os.path.join(CSRC, "loop_verify_submap.cu")]
GMD_LIB = os.path.join(HERE, "libtloam_b200_gmd.so")
GMD_SOURCES = [os.path.join(CSRC, "map_dynamic.cu")]
GMM_LIB = os.path.join(HERE, "libtloam_b200_gmm.so")
GMM_SOURCES = [os.path.join(CSRC, "map_merge.cu")]
LOC_LIB = os.path.join(HERE, "libtloam_b200_loc.so")
LOC_SOURCES = [os.path.join(CSRC, "localize.cu")]
RELOC_LIB = os.path.join(HERE, "libtloam_b200_reloc.so")
RELOC_SOURCES = [os.path.join(CSRC, "relocalize.cu")]
MAPU_LIB = os.path.join(HERE, "libtloam_b200_mapu.so")
MAPU_SOURCES = [os.path.join(CSRC, "map_update.cu")]
OCC_LIB = os.path.join(HERE, "libtloam_b200_occ.so")
OCC_SOURCES = [os.path.join(CSRC, "occupancy.cu")]
DIST_LIB = os.path.join(HERE, "libtloam_b200_dist.so")
DIST_SOURCES = [os.path.join(CSRC, "distance.cu")]
PLAN_LIB = os.path.join(HERE, "libtloam_b200_plan.so")
PLAN_SOURCES = [os.path.join(CSRC, "plan.cu")]
GREG_LIB = os.path.join(HERE, "libtloam_b200_greg.so")
GREG_SOURCES = [os.path.join(CSRC, "global_registration.cu")]
FRONTIER_LIB = os.path.join(HERE, "libtloam_b200_frontier.so")
FRONTIER_SOURCES = [os.path.join(CSRC, "frontier.cu")]
TERRAIN_LIB = os.path.join(HERE, "libtloam_b200_terrain.so")
TERRAIN_SOURCES = [os.path.join(CSRC, "terrain.cu")]
import glob
# every header the translation unit can include: editing any of them triggers a rebuild
HEADERS = sorted(glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) +
                 glob.glob(os.path.join(HERE, "..", "include", "**", "*.h"), recursive=True))

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "static", "-ccbin", "/usr/bin/g++",
]


def needs_build(lib=LIB, sources=SOURCES):
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    return any(os.path.getmtime(p) > t for p in sources + HEADERS + [os.path.abspath(__file__)])


def _nvcc(lib, sources, verbose, extra):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + list(extra) + ["-o", lib] + sources
    if verbose:
        print(" ".join(cmd))
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose and (res.stdout or res.stderr):
        print(res.stdout + res.stderr)


def build(force=False, verbose=False, extra=()):
    """builds the twenty-one libraries (each only when out of date); returns the path of libtloam_b200.so"""
    for lib, sources in ((LIB, SOURCES), (GMI_LIB, GMI_SOURCES), (UNPACK_LIB, UNPACK_SOURCES), (DESKEW_LIB, DESKEW_SOURCES),
                         (LOOP_LIB, LOOP_SOURCES), (LOOPV_LIB, LOOPV_SOURCES), (PG_LIB, PG_SOURCES), (GMC_LIB, GMC_SOURCES),
                         (PGR_LIB, PGR_SOURCES), (LOOPVS_LIB, LOOPVS_SOURCES), (GMD_LIB, GMD_SOURCES),
                         (GMM_LIB, GMM_SOURCES), (LOC_LIB, LOC_SOURCES), (RELOC_LIB, RELOC_SOURCES),
                         (MAPU_LIB, MAPU_SOURCES), (OCC_LIB, OCC_SOURCES), (DIST_LIB, DIST_SOURCES),
                         (PLAN_LIB, PLAN_SOURCES), (GREG_LIB, GREG_SOURCES), (FRONTIER_LIB, FRONTIER_SOURCES),
                         (TERRAIN_LIB, TERRAIN_SOURCES)):
        if force or needs_build(lib, sources):
            _nvcc(lib, sources, verbose, extra)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True,
                extra=("-Xptxas", "-v") if "--ptxas" in sys.argv else ()))
