"""`python -m cape_b200.main --config configs/<x>.yaml --mode train ...`: the reference's main.py (main.py:1-113) on
the H100 engine.

Same flow: parse the config (the reference's yaml files load unchanged), load the dataset (`BodyData`), build the mesh
hierarchy for `--num_conv_layers` / `--ds_factor`, construct `CAPE` and train.  The hierarchy is GENERATED from the
template mesh like main.py:38 does (cape_b200.mesh_sampling: no psbody); for the default 8 layers / factor 2 that
reproduces the reference's shipped `for_demo` fixtures exactly, so a model trained here is the model the demo scripts load.
The discriminator keeps the pre-computed `ds2` hierarchy (main.py:46).  `--mode test` and `--mode demo` build the model
for the demo phase on the same hierarchy, restore its checkpoint and run `demos.demo_full` (main.py:101-109): the test
mode measures the auto-encoding error of the test set, the demo mode generates clothing under six poses and four
clothing types; both pose their meshes with the SMPL model `<smpl_model_folder>/smpl/SMPL_<GENDER>.pkl` on the GPU.
The on-screen viewers of `--vis_demo 1` are not available.  The clothing-generation demo without posing is
`python -m cape_b200.demos` (= run_simple_demo.py).
"""
import os

import numpy as np

from . import mesh_sampling, topology
from .config_parser import model_params, parse_config
from .demos import demo_full
from .load_data import BodyData
from .models import CAPE


def build_hierarchy(num_conv_layers=8, ds_factor=2, mesh=None):
    """(L, D, U, p) of the VAE for main.py:31-43.  mesh: anything with .v / .f (default: the SMPL template)."""
    if mesh is None:
        v, f = topology.template_mesh()
        mesh = mesh_sampling.TriMesh(v=v, f=f)
    return mesh_sampling.hierarchy(mesh, num_conv_layers, ds_factor)


def main(argv=None, project_dir=None):
    args, args_dict = parse_config(argv)
    np.random.seed(args_dict["seed"])
    project_dir = project_dir or os.environ.get("CAPE_REFERENCE") or os.getcwd()
    data_dir = os.path.join(project_dir, "data", "datasets", args.dataset)
    if args.mode == "demo":
        bodydata = None
    else:
        print("Loading data from {} ..".format(data_dir))
        bodydata = load_body_data(data_dir, args.pose_type)
    print("Pre-computing mesh pooling matrices ..")
    L, D, U, p = build_hierarchy(args.num_conv_layers, args.ds_factor)
    L_ds2, D_ds2, _ = topology.load_graph_mtx()
    params = model_params(args, n_train=len(bodydata.vertices_train) if args.mode == "train" else None)
    params["p"] = p
    print("Building model graph...")
    # training writes TensorBoard summaries to summaries/<name>, relative to the working directory like checkpoints/
    model = CAPE(L=L, D=D, U=U, L_d=L_ds2, D_d=D_ds2, summary_dir="summaries" if args.mode == "train" else None, **params)
    if args.mode == "train":
        model.build_graph(model.input_num_verts, model.nn_input_channel, phase="train")
        return model.fit(bodydata)
    model.build_graph(model.input_num_verts, model.nn_input_channel, phase="demo")
    demos = demo_full(model, args.name, args.gender, args.dataset, data_dir, os.path.dirname(data_dir),
                      n_sample=args.demo_n_sample, save_obj=bool(args.save_obj), random_seed=args.seed,
                      vis=bool(args.vis_demo), smpl_model_folder=os.path.join(project_dir, args.smpl_model_folder),
                      results_dir=os.path.join(project_dir, "results", args.name))
    if args.mode == "test":
        return demos.test_model(bodydata)
    return demos.run()


def load_body_data(data_dir, pose_type):
    """The dataset as main.py:20-29 loads it."""
    return BodyData(nVal=100,
                    train_mesh_fn=data_dir + "/train/train_disp.npy",
                    train_cond1_fn=data_dir + "/train/train_{}.npy".format(pose_type),
                    train_cond2_fn=data_dir + "/train/train_{}.npy".format("clo_label"),
                    test_mesh_fn=data_dir + "/test/test_disp.npy",
                    test_cond1_fn=data_dir + "/test/test_{}.npy".format(pose_type),
                    test_cond2_fn=data_dir + "/test/test_{}.npy".format("clo_label"))


if __name__ == "__main__":
    main()
