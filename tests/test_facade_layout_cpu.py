"""The facade's pipeline header has the reference's shape (VERDICT r1 #5): ONE translation unit is compiled twice — against
the reference's own pipeline/KinematicICP.hpp (with the oracle's header shims for the libraries that are absent offline) and
against this repo's facade header — using aggregate initialisation of Config, assignment of every field by name and a
subclass that reaches the five protected members by name; the two builds must report the same sizeof / offsetof of Config.
The facade build is always checked against the numbers recorded from the reference build; the reference header itself is
compiled too when KICP_REFERENCE_DIR names a reference checkout."""
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(os.environ.get("KICP_REFERENCE_DIR", ""), "cpp")
TU = r"""
#include <cstddef>
#include <cstdio>
#include "kinematic_icp/pipeline/KinematicICP.hpp"
using namespace kinematic_icp::pipeline;
struct Probe : KinematicICP {  // a subclass touching the protected members by the reference's names
    using KinematicICP::KinematicICP;
    void poke() {
        (void)sizeof(registration_.max_num_iterations_);
        (void)sizeof(correspondence_threshold_.odom_sse_);
        (void)sizeof(config_.voxel_size);
        (void)sizeof(preprocessor_);
        (void)sizeof(local_map_);
        (void)sizeof(last_pose_);
    }
};
int main() {
    // aggregate initialisation in declaration order (pipeline/KinematicICP.hpp:38-60)
    Config c{80.0, 0.5, 0.75, 12u, false, 2.0, 7, 1e-4, 3, false, 0.25, true};
    if (c.max_range != 80.0 || c.min_range != 0.5 || c.voxel_size != 0.75 || c.max_points_per_voxel != 12u ||
        c.use_adaptive_threshold || c.fixed_threshold != 2.0 || c.max_num_iterations != 7 || c.convergence_criterion != 1e-4 ||
        c.max_num_threads != 3 || c.use_adaptive_odometry_regularization || c.fixed_regularization != 0.25 || !c.deskew)
        return 1;
    Config d;  // defaults
    if (d.max_range != 100.0 || d.voxel_size != 1.0 || d.max_points_per_voxel != 20u || !d.use_adaptive_threshold ||
        d.max_num_iterations != 10 || d.convergence_criterion != 0.001 || d.max_num_threads != 1 ||
        !d.use_adaptive_odometry_regularization || d.fixed_regularization != 0.0 || d.deskew)
        return 2;
    printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(Config), offsetof(Config, max_range), offsetof(Config, min_range),
           offsetof(Config, voxel_size), offsetof(Config, max_points_per_voxel), offsetof(Config, use_adaptive_threshold),
           offsetof(Config, fixed_threshold), offsetof(Config, max_num_iterations), offsetof(Config, convergence_criterion),
           offsetof(Config, max_num_threads), offsetof(Config, use_adaptive_odometry_regularization),
           offsetof(Config, fixed_regularization), offsetof(Config, deskew));
    return 0;
}
"""
EXPECTED = "80 0 8 16 24 28 32 40 48 56 60 64 72"  # the reference's layout on x86-64 (recorded from the reference build)


def compile_tu(includes, defines=()):
    """Compile the full TU (subclass included) to an object file, then build + run a link-free variant that prints the layout."""
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "tu.cpp")
        open(src, "w").write(TU)
        inc = ["-I" + i for i in includes]
        r = subprocess.run(["g++", "-std=c++17", "-O0", "-c", "-o", os.path.join(d, "tu.o")] + inc + list(defines) + [src],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        # layout: same headers, only Config is used -> nothing to link
        lay = os.path.join(d, "lay.cpp")
        body = TU[TU.index("int main() {"):]
        open(lay, "w").write('#include <cstddef>\n#include <cstdio>\n#include "kinematic_icp/pipeline/KinematicICP.hpp"\n'
                             "using namespace kinematic_icp::pipeline;\n" + body)
        r = subprocess.run(["g++", "-std=c++17", "-O0", "-o", os.path.join(d, "lay")] + inc + list(defines) + [lay, "-Wl,--unresolved-symbols=ignore-all"],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        out = subprocess.run([os.path.join(d, "lay")], capture_output=True, text=True)
        assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
        return out.stdout.strip()


def test_facade_config_and_members_match_the_reference_header():
    facade_inc = [os.path.join(ROOT, "kinematic-icp_b200", "cpp"), os.path.join(ROOT, "kinematic-icp_b200", "cpp", "compat"),
                  os.path.join(ROOT, "include")]
    got = compile_tu(facade_inc)
    assert got == EXPECTED, got
    if os.path.isdir(os.path.join(REF, "kinematic_icp")):
        ref_inc = [REF, os.path.join(ROOT, "oracle", "shim"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "kinematic-icp_b200", "cpp", "compat")]
        ref = compile_tu(ref_inc)
        assert ref == got == EXPECTED, (ref, got)
