"""`demo_simple`: the reference's clothing-generation demo (demos.py:339-406, run_simple_demo.py) on the H100 engine.

Fix a body pose, run the four clothing types through the condition nets, draw latent codes, decode
(`CAPE.decode`: decoder-only generation, the latency-sensitive serving path), de-normalise with the training-set
statistics, keep the clothing-related vertices only, add the minimal body shape and write OBJ files.  No trimesh /
psbody / smplx: meshes are written by a ten-line OBJ writer, everything else is numpy around the model API.
"""
import os

import numpy as np

from . import topology as topo

# indices of the SMPL joints related to clothing (lib/utils.py:38)
useful_joints_idx = [1, 2, 3, 4, 5, 6, 9, 12, 13, 14, 16, 17, 18, 19]


def filter_cloth_pose(pose_vec):
    """72-dim pose vectors or 216-dim rotation matrices -> the 14 clothing-related joints (lib/utils.py:40-62)."""
    pose_vec = np.asarray(pose_vec)
    n, dim = pose_vec.shape[0], pose_vec.shape[-1]
    if dim == 72:
        arr = pose_vec.reshape(n, -1, 3)
    elif dim == 216:
        arr = pose_vec.reshape(n, -1, 9)
    else:
        raise ValueError("please provide either 72-dim pose vector or 216-dim rot matrix")
    return arr[:, useful_joints_idx, :].reshape(n, -1)


def write_obj(path, vertices, faces):
    with open(path, "w") as f:
        for v in np.asarray(vertices, np.float64):
            f.write("v %.8f %.8f %.8f\n" % (v[0], v[1], v[2]))
        for t in np.asarray(faces) + 1:
            f.write("f %d %d %d\n" % (t[0], t[1], t[2]))


def read_obj(path):
    v, f = [], []
    for ln in open(path):
        t = ln.split()
        if t and t[0] == "v":
            v.append([float(x) for x in t[1:4]])
        elif t and t[0] == "f":
            f.append([int(x.split("/")[0]) - 1 for x in t[1:4]])
    return np.asarray(v), np.asarray(f, np.int32)


class demo_simple(object):
    """Same constructor and method as the reference's class (demos.py:339-406); `results_dir` and `n_sample` may be
    overridden, `sample_vary_clotype` additionally returns {clothing type: [n_sample, 6890, 3] full-body vertices}."""

    def __init__(self, model, name, random_seed=123, results_dir=None, n_sample=3, save_obj=True):
        self.name, self.model = name, model
        self.n_sample, self.save_obj = n_sample, save_obj
        self.clo_type_readable = np.array(["shortlong", "shortshort", "longshort", "longlong"])
        self.clothing_verts_idx = topo.clothing_verts_idx()
        self.minimal_shape, self.faces = topo.template_mesh()
        self.rot, self.pose = topo.demo_pose_params()
        self.train_mean, self.train_std = topo.trainset_stats()
        self.results_dir = results_dir or os.path.join(os.getcwd(), "results", "demo_results")
        os.makedirs(self.results_dir, exist_ok=True)
        np.random.seed(random_seed)

    def postprocess(self, predictions):
        """Network output -> full-body vertices (demos.py:394-402): de-normalise, zero the displacements of head,
        fingers and toes, add the minimal body shape."""
        predictions = predictions * self.train_std + self.train_mean
        disp_masked = np.zeros_like(predictions)
        disp_masked[:, self.clothing_verts_idx, :] = predictions[:, self.clothing_verts_idx, :]
        return disp_masked + self.minimal_shape

    def sample_vary_clotype(self):
        """fix body pose, sample 4 clothing types, under each clothing type sample latent code N times"""
        clotype = np.eye(4, dtype=np.float32)
        rot = filter_cloth_pose(self.rot)[0]
        rot_repeated = np.repeat(rot[np.newaxis, :], len(clotype), axis=0).astype(np.float32)
        pose_emb, clotype_emb = self.model.encode_only_condition(rot_repeated, clotype)
        pose_emb = pose_emb[0]
        print("\n=============== Running demo: fix z, pose, change clothing type ===============")
        print("Found {} different clothing types, for each we generate {} samples\n".format(len(clotype), self.n_sample))
        z_samples = np.random.normal(loc=0.0, scale=1.0, size=(self.n_sample, self.model.nz))
        out = {}
        for i in range(len(clotype)):
            clotype_emb_i = clotype_emb[i]
            clotype_name = self.clo_type_readable[np.argmax(clotype[i])]
            z_sample_c = np.array([np.concatenate([s.reshape(1, -1), pose_emb.reshape(1, -1), clotype_emb_i.reshape(1, -1)],
                                                  axis=1) for s in z_samples]).reshape(self.n_sample, -1)
            predictions = self.model.decode(z_sample_c.astype(np.float32), cond=pose_emb.reshape(1, -1),
                                            cond2=clotype_emb_i.reshape(1, -1))
            full = self.postprocess(predictions)
            out[str(clotype_name)] = full
            if self.save_obj:
                for j in range(self.n_sample):
                    write_obj(os.path.join(self.results_dir, "{}_{:0>4d}.obj".format(clotype_name, j)), full[j], self.faces)
        return out


def run_simple_demo(argv=None):
    """run_simple_demo.py: parse the config, build the model, restore its checkpoint, write the demo meshes."""
    from .config_parser import model_params, parse_config
    from .models import CAPE
    args, args_dict = parse_config(argv)
    np.random.seed(args_dict["seed"])
    L, D, U, p, L_ds2, D_ds2, _ = topo.load_graph_mtx(load_for_demo=True)
    params = model_params(args)
    params["p"] = p
    model = CAPE(L=L, D=D, U=U, L_d=L_ds2, D_d=D_ds2, **params)
    model.build_graph(model.input_num_verts, model.nn_input_channel, phase="demo")
    demo = demo_simple(model, args.name, args.seed)
    return demo.sample_vary_clotype()


if __name__ == "__main__":
    run_simple_demo()
