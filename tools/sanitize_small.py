"""Every entry point once on small inputs -- meant to run under compute-sanitizer:
   compute-sanitizer --tool memcheck  python tools/sanitize_small.py
   compute-sanitizer --tool racecheck python tools/sanitize_small.py
   compute-sanitizer --tool initcheck python tools/sanitize_small.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import pcu_b200 as pcu

rng = np.random.default_rng(0)
n = int(sys.argv[1]) if len(sys.argv) > 1 else 6000
x = rng.random((n, 3)).astype(np.float32)
y = rng.random((n + 137, 3)).astype(np.float32)
lat = np.stack(np.meshgrid(*[np.arange(12)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32) / 12   # ties everywhere


def step(name, fn):
    out = fn()
    torch.cuda.synchronize()
    print("ok", name, flush=True)
    return out


step("knn k=1", lambda: pcu.k_nearest_neighbors(x, y, 1))
step("knn k=16", lambda: pcu.k_nearest_neighbors(x, y, 16))
step("knn k=5 fp64", lambda: pcu.k_nearest_neighbors(x.astype(np.float64), y.astype(np.float64), 5))
step("knn k=40 (pyramid path)", lambda: pcu.k_nearest_neighbors(x[:2000], y, 40))
step("knn lattice k=8 (tie replay)", lambda: pcu.k_nearest_neighbors(lat + 0.01, lat, 8))
step("knn far apart", lambda: pcu.k_nearest_neighbors(x + 50.0, y, 4))
step("knn tiny clouds (one-CTA binning)", lambda: pcu.k_nearest_neighbors(x[:300], y[:200], 3))
step("chamfer", lambda: pcu.chamfer_distance(x, y))
step("chamfer return_index", lambda: pcu.chamfer_distance(x, y, return_index=True))
step("hausdorff", lambda: pcu.hausdorff_distance(x, y, return_index=True))
step("hausdorff lattice (witness replay)", lambda: pcu.hausdorff_distance(lat + 0.5 / 12, lat, return_index=True))
step("one-sided hausdorff fp64", lambda: pcu.one_sided_hausdorff_distance(x.astype(np.float64), y.astype(np.float64)))
xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
step("device tensors chamfer", lambda: float(pcu.chamfer_distance(xt, yt)))
step("batched chamfer", lambda: pcu.batched_chamfer_distance(rng.random((6, 900, 3), dtype=np.float32), rng.random((6, 1100, 3), dtype=np.float32)))
step("batched chamfer (grid-wide binning)", lambda: pcu.batched_chamfer_distance(rng.random((2, 9000, 3), dtype=np.float32), rng.random((2, 9100, 3), dtype=np.float32)))
prep = step("prepare_cloud", lambda: pcu.prepare_cloud(y))
step("chamfer against a prepared cloud", lambda: pcu.chamfer_distance(x, prep))
step("hausdorff against a prepared cloud", lambda: pcu.one_sided_hausdorff_distance(x, prep))
v = rng.normal(size=(n, 3)); v /= np.linalg.norm(v, axis=1, keepdims=True)
step("normals knn", lambda: pcu.estimate_point_cloud_normals_knn(v.astype(np.float32), 10, v.astype(np.float32), np.deg2rad(30)))
step("normals ball", lambda: pcu.estimate_point_cloud_normals_ball(v.astype(np.float32), 0.01, v.astype(np.float32), np.deg2rad(30), 5, weight_function="rbf"))
step("normals ball, capped, fp64", lambda: pcu.estimate_point_cloud_normals_ball(v, 0.01, max_pts_per_ball=6))
step("voxel down-sampling", lambda: pcu.downsample_point_cloud_on_voxel_grid(0.05, x, x.astype(np.float64)))
step("deduplicate points", lambda: pcu.deduplicate_point_cloud(np.concatenate([x, x[:500]]), 1e-6))
step("deduplicate mesh fp64", lambda: pcu.deduplicate_mesh_vertices(np.concatenate([x, x[:500]]).astype(np.float64), rng.integers(0, n, (3000, 3)).astype(np.int64), 0.0))
mv = rng.normal(size=(200, 3)); mf = rng.integers(0, 200, (300, 3))
ro = rng.normal(size=(500, 3)) * 3
step("ray mesh intersection", lambda: pcu.ray_mesh_intersection(mv, mf, ro, -ro))
step("ray mesh intersection, one origin fp32", lambda: pcu.ray_mesh_intersection(mv.astype(np.float32), mf, np.zeros(3, np.float32), ro.astype(np.float32)))
isect = step("prepare a mesh for rays", lambda: pcu.RayMeshIntersector(mv.astype(np.float32), mf))
step("rays against a prepared mesh (fp64 rays)", lambda: isect.intersect_rays(ro, -ro))
isect.close()
sp, sn = rng.normal(size=(300, 3)), rng.normal(size=(300, 3))
step("ray surfel intersection", lambda: pcu.ray_surfel_intersection(sp, sn, ro, -ro, 0.3, 7))
step("surfel geometry fp32", lambda: pcu.pointcloud_surfel_geometry(sp.astype(np.float32), sn.astype(np.float32), 0.3, 5))
surf = step("prepare surfels for rays", lambda: pcu.RaySurfelIntersector(sp.astype(np.float32), sn.astype(np.float32), 0.3))
step("rays against prepared surfels (fp64 rays)", lambda: surf.intersect_rays(ro, -ro))
surf.close()
cn = rng.normal(size=(n, 3)); ca = rng.random(n)
step("point cloud winding numbers", lambda: pcu.point_cloud_fast_winding_number(v, cn, ca, ro))
step("point cloud winding numbers fp32", lambda: pcu.point_cloud_fast_winding_number(v.astype(np.float32), cn.astype(np.float32), ca.astype(np.float32), ro.astype(np.float32)))
ax = np.linspace(-1, 1, 12)
gz, gy, gx = np.meshgrid(ax, ax, ax, indexing="ij")
gc = np.stack([gx.ravel(), gy.ravel(), gz.ravel()], 1)
cb = np.arange(12 ** 3).reshape(12, 12, 12)[:-1, :-1, :-1].ravel()[:, None] + np.array([0, 1, 13, 12, 144, 145, 157, 156])
step("marching cubes", lambda: pcu.marching_cubes_sparse_voxel_grid(np.linalg.norm(gc, axis=1) - 0.6, gc, cb, 0.0))
step("marching cubes fp32 / uint32", lambda: pcu.marching_cubes_sparse_voxel_grid(
    (np.linalg.norm(gc, axis=1) - 0.6).astype(np.float32), gc.astype(np.float32), cb.astype(np.uint32), 0.0))
tf = np.concatenate([mf[:, :2], mf[:, :2] + 205, rng.integers(0, 60, (40, 2)) + 400])
step("connected components", lambda: pcu.connected_components(mv, np.concatenate([mf, mf + 205])))
step("connected components uint64 edges", lambda: pcu.connected_components(mv.astype(np.float32), tf.astype(np.uint64)))
step("remove mesh vertices", lambda: pcu.remove_mesh_vertices(mv, mf, rng.random(200) < 0.7))
step("remove unreferenced vertices fp32 / uint32", lambda: pcu.remove_unreferenced_mesh_vertices(mv.astype(np.float32), mf[:50].astype(np.uint32)))
step("orient mesh faces", lambda: pcu.orient_mesh_faces(np.concatenate([mf, mf[::-1, ::-1] + 205])))
step("orient mesh faces uint64, repeated corners (replayed)", lambda: pcu.orient_mesh_faces(rng.integers(0, 12, (60, 3)).astype(np.uint64)))
step("mesh face areas", lambda: pcu.mesh_face_areas(mv, mf))
step("face normals fp32 / uint32", lambda: pcu.estimate_mesh_face_normals(mv.astype(np.float32), mf.astype(np.uint32)))
step("vertex normals area", lambda: pcu.estimate_mesh_vertex_normals(mv, mf, "area"))
step("vertex normals angle fp32", lambda: pcu.estimate_mesh_vertex_normals(mv.astype(np.float32), mf.astype(np.int32), "angle"))
step("laplacian smoothing", lambda: pcu.laplacian_smooth_mesh(mv, mf, 2))
step("laplacian smoothing cotan fp32", lambda: pcu.laplacian_smooth_mesh(mv.astype(np.float32), mf.astype(np.int32), 2, use_cotan_weights=True))
step("sparse voxel grid boundary",lambda: pcu.sparse_voxel_grid_boundary(rng.integers(-10, 10, (n, 3)).astype(np.int32)))
pts_i = rng.integers(-1000, 1000, (n, 3)).astype(np.int32)
codes = step("morton encode", lambda: pcu.morton_encode(pts_i))
step("morton decode", lambda: pcu.morton_decode(codes))
step("morton add", lambda: pcu.morton_add(codes, codes))
step("morton knn", lambda: pcu.morton_knn(np.sort(codes), codes[:500], 7))
a = rng.random((40, 3)); b = rng.random((50, 3))
M = step("pairwise distances", lambda: pcu.pairwise_distances(a, b))
step("sinkhorn", lambda: pcu.sinkhorn(np.full(40, 1 / 40), np.full(50, 1 / 50), M, eps=1e-2, max_iters=50))
step("earth mover's distance", lambda: pcu.earth_movers_distance(a, b, eps=1e-2, max_iters=50))
print("done")
