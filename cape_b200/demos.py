"""`demo_simple`: the reference's clothing-generation demo (demos.py:339-406, run_simple_demo.py) on the H100 engine.

Fix a body pose, run the four clothing types through the condition nets, draw latent codes, decode
(`CAPE.decode`: decoder-only generation, the latency-sensitive serving path), de-normalise with the training-set
statistics, keep the clothing-related vertices only, add the minimal body shape and write OBJ files.  No trimesh /
psbody / smplx: meshes are written by a ten-line OBJ writer, everything else is numpy around the model API.

`demo_full`: the reference's test / demo modes (demos.py:9-336): the same flow for six poses and four clothing types,
plus the auto-encoding error of a test set, with every mesh posed by the SMPL body model on the GPU (cape_b200.smpl).
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


def postprocess(predictions, mean, std, clothing_verts_idx, minimal_shape):
    """Network output -> full-body vertices (demos.py:394-402): de-normalise, zero the displacements of head,
    fingers and toes, add the minimal body shape."""
    predictions = predictions * std + mean
    disp_masked = np.zeros_like(predictions)
    disp_masked[:, clothing_verts_idx, :] = predictions[:, clothing_verts_idx, :]
    return disp_masked + minimal_shape


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
        return postprocess(predictions, self.train_mean, self.train_std, self.clothing_verts_idx, self.minimal_shape)

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


class demo_full(object):
    """The reference's test / demo modes (demos.py:9-336): `test_model` (auto-encoding error over the clothing vertices
    of the test set, posed exemplars), `sample_vary_pose`, `sample_vary_clotype` and `run`.  Generated clothing is posed
    with the SMPL body model on the GPU (cape_b200.smpl) instead of smplx.  Same constructor; additionally
    `body_model` (anything with `faces` and `pose(verts [N, V, 3], pose [N, 72]) -> verts`; default: the SMPL pickle
    of `gender` under `smpl_model_folder`) and `results_dir` (default: ./results/<name>).  The methods return what
    they pose.  The psbody viewers (`vis`) are not available: their meshes are neither posed nor shown."""

    def __init__(self, model, name, gender, dataset, data_dir, datadir_root, n_sample, save_obj,
                 smpl_model_folder="body_models", random_seed=123, vis=True, body_model=None, results_dir=None):
        self.n_sample, self.name, self.model, self.dataset = n_sample, name, model, dataset
        self.data_dir, self.datadir_root = data_dir, datadir_root
        self.save_obj, self.vis = save_obj, vis
        if vis:
            print("vis_demo: the on-screen mesh viewer is not available, continuing without it")
        if body_model is None:
            from .smpl import SMPL, model_path
            body_model = SMPL(model_path(smpl_model_folder, gender))
        self.body_model = body_model
        self.clo_type_readable = np.array(["shortlong", "shortshort", "longshort", "longlong"])
        self.clothing_verts_idx = topo.clothing_verts_idx()
        self.minimal_shape, _ = topo.template_mesh()
        self.rot, self.pose = topo.demo_pose_params()
        self.train_mean, self.train_std = topo.trainset_stats()
        self.results_dir = results_dir or os.path.join(os.getcwd(), "results", name)
        os.makedirs(self.results_dir, exist_ok=True)
        np.random.seed(random_seed)

    def postprocess(self, predictions, mean=None, std=None):
        """postprocess() with the training-set statistics unless others are given."""
        return postprocess(predictions, self.train_mean if mean is None else mean,
                           self.train_std if std is None else std, self.clothing_verts_idx, self.minimal_shape)

    def pose_and_save(self, verts, poses, obj_dir, pattern):
        """Pose every mesh with its pose (demos.py:249-331) and, with save_obj, write obj_dir/pattern.format(i)."""
        posed = self.body_model.pose(np.asarray(verts), np.asarray(poses))
        if self.save_obj:
            os.makedirs(obj_dir, exist_ok=True)
            print("saving results as .obj files to {}...".format(obj_dir))
            for i, v in enumerate(posed):
                write_obj(os.path.join(obj_dir, pattern.format(i)), v, self.body_model.faces)
        return posed

    def test_model(self, bodydata):
        """Auto-encoding error of the test set (demos.py:47-124).  Returns {'string', 'mean', 'std', 'median',
        'posed'}; 'posed' holds the posed exemplars (None without `cond1_test_full` or save_obj)."""
        print("\n=============== Running demo: test reconstruction ===============")
        obj_dir = os.path.join(self.results_dir, "test_reconstruction_objs_{}".format(self.dataset))
        vertices = bodydata.vertices_test
        print("\nTesting on test set, {} examples...\n".format(len(vertices)))
        predictions, recon_loss, latent_loss, edge_loss = self.model.predict(data=vertices, cond=bodydata.cond1_test,
                                                                             cond2=bodydata.cond2_test, labels=vertices,
                                                                             phase="test")
        predictions = predictions * bodydata.std + bodydata.mean
        gt = vertices * bodydata.std + bodydata.mean
        diff = (predictions - gt)[:, self.clothing_verts_idx, :]
        err = np.sqrt(np.sum(diff ** 2, axis=2))
        mean, std, median = np.mean(err), np.std(err), np.median(err)
        test_result_str = "\nResults from {}: \n" \
                          "L1 {:.5f}, KL {:.5f}, Edge {:.5f}\n" \
                          "Eucledian err mean {:.5f}, std {:.5f}, median {:.5f}.\n".format(self.name,
                                recon_loss, latent_loss, edge_loss, mean, std, median)
        print(test_result_str)
        for fn in (os.path.join(self.results_dir, "test_results_{}.txt".format(self.dataset)),
                   os.path.join(self.results_dir, "..", "all_test_results_{}.txt".format(self.dataset))):
            with open(fn, "a+") as fp:
                fp.write(test_result_str)
        posed = None
        if self.save_obj and hasattr(bodydata, "cond1_test_full"):
            predictions_fullbody = self.postprocess(predictions, mean=0.0, std=1.0)
            pose_full = bodydata.cond1_test_full
            if pose_full.shape[-1] == 216:            # rotation-matrix conditions -> axis-angle poses
                from .smpl import rot2pose
                pose_full = rot2pose(pose_full)
            step = int(len(gt) / self.n_sample)        # exemplars only; the stride may give more than n_sample
            posed = self.pose_and_save(predictions_fullbody[::step], pose_full[::step], obj_dir, "{:0>4d}.obj")
        return {"string": test_result_str, "mean": mean, "std": std, "median": median, "posed": posed}

    def _decode(self, z_samples, pose_emb, clotype_emb):
        z_sample_c = np.array([np.concatenate([s.reshape(1, -1), pose_emb.reshape(1, -1), clotype_emb.reshape(1, -1)],
                                              axis=1) for s in z_samples]).reshape(self.n_sample, -1)
        return self.model.decode(z_sample_c.astype(np.float32), cond=pose_emb.reshape(1, -1),
                                 cond2=clotype_emb.reshape(1, -1))

    def sample_vary_pose(self):
        """fix clothing type, sample several poses, under each pose sample latent code N times (demos.py:127-169).
        Returns [len(poses)] arrays of posed meshes [n_sample, V, 3]."""
        rot = filter_cloth_pose(self.rot)
        clotype = (self.clo_type_readable == "shortlong").astype(np.float32)
        clotype_repeated = np.repeat(clotype[np.newaxis, :], len(rot), axis=0)
        pose_emb, clotype_emb = self.model.encode_only_condition(rot.astype(np.float32), clotype_repeated)
        clotype_emb = clotype_emb[0]
        obj_dir = os.path.join(self.results_dir, "sample_vary_pose")
        print("\n=============== Running demo: fix z, clotype, change pose ===============")
        print("\nFound {} different pose, for each we generate {} samples\n".format(len(rot), self.n_sample))
        z_samples = np.random.normal(loc=0.0, scale=1.0, size=(self.n_sample, self.model.nz))
        out = []
        for idx, pose_emb_i in enumerate(pose_emb):
            full = self.postprocess(self._decode(z_samples, pose_emb_i, clotype_emb))
            poses = np.repeat(self.pose[np.newaxis, idx, :], self.n_sample, axis=0)
            out.append(self.pose_and_save(full, poses, obj_dir, "pose%d_{:0>4d}.obj" % idx))
        return out

    def sample_vary_clotype(self):
        """fix body pose, sample 4 clothing types, under each clothing type sample latent code N times
        (demos.py:172-246).  As in the reference, the clothing is generated for the condition of demo pose 0 and posed
        with demo pose 2.  Returns {clothing type: posed meshes [n_sample, V, 3]}."""
        poses = np.repeat(self.pose[np.newaxis, 2], self.n_sample, axis=0)
        clotype = np.eye(4, dtype=np.float32)
        rot = filter_cloth_pose(self.rot)[0]
        rot_repeated = np.repeat(rot[np.newaxis, :], len(clotype), axis=0).astype(np.float32)
        pose_emb, clotype_emb = self.model.encode_only_condition(rot_repeated, clotype)
        pose_emb = pose_emb[0]
        print("\n=============== Running demo: fix z, pose, change clothing type ===============")
        print("Found {} different clothing types, for each we generate {} samples\n".format(len(clotype), self.n_sample))
        obj_dir = os.path.join(self.results_dir, "sample_vary_clotype")
        z_samples = np.random.normal(loc=0.0, scale=1.0, size=(self.n_sample, self.model.nz))
        out = {}
        for i in range(len(clotype)):
            name = str(self.clo_type_readable[np.argmax(clotype[i])])
            full = self.postprocess(self._decode(z_samples, pose_emb, clotype_emb[i]))
            out[name] = self.pose_and_save(full, poses, obj_dir, "clotype_%s_{:0>4d}.obj" % name)
        return out

    def run(self):
        return self.sample_vary_pose(), self.sample_vary_clotype()


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
