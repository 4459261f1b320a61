"""The drop-in launcher under torch.multiprocessing.spawn (no GPU needed).

`main.py` starts one process per GPU with torch.multiprocessing.spawn (main.py:1103-1120).  The children must import
the package's `models`, `criterion` and `third_party_pointnet2` shims, not the modules of the checkout that lie next to
the script.  The checkout here is a directory whose modules of those names raise on import."""
import json
import os
import subprocess
import sys
import textwrap
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
PACKAGE = ROOT / "coda_neurips2023_b200"

SCRIPT = textwrap.dedent('''
    import json
    import os
    import sys

    import torch.multiprocessing as mp


    def child(rank, outdir):
        import warnings

        import torch

        import criterion
        import models
        import third_party_pointnet2.pointnet2.pointnet2_modules as pm
        from coda_neurips2023_b200 import synthetic

        args = synthetic.make_args(nqueries=128, preenc_npoints=256, dec_dim=128, dec_nlayers=2, dec_ffn_dim=64)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model, _ = models.build_model(args, synthetic.SyntheticDatasetConfig(args))
        plain = list(model.state_dict())
        converted = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
        nsync = sum(isinstance(m, torch.nn.SyncBatchNorm) for m in converted.modules())
        with open(os.path.join(outdir, "rank%d.json" % rank), "w") as f:
            json.dump({"models": models.__file__, "criterion": criterion.__file__, "pointnet2_modules": pm.__file__,
                       "plain_keys": plain, "converted_keys": list(converted.state_dict()), "nsync": nsync}, f)


    if __name__ == "__main__":
        mp.set_start_method("spawn", force=True)
        mp.spawn(child, nprocs=2, args=(sys.argv[1],), join=True)
''')


def test_spawned_children_import_the_package_shims(tmp_path):
    checkout = tmp_path / "checkout"
    for rel in ("models/__init__.py", "criterion.py", "third_party_pointnet2/__init__.py",
                "third_party_pointnet2/pointnet2/__init__.py", "third_party_pointnet2/pointnet2/pointnet2_modules.py"):
        f = checkout / rel
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_text(f"raise ImportError('the checkout\\'s {rel} was imported')\n")
    (checkout / "main.py").write_text(SCRIPT)
    out = tmp_path / "out"
    out.mkdir()
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(ROOT)] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    r = subprocess.run([sys.executable, "-m", "coda_neurips2023_b200.dropin.launch", str(checkout / "main.py"),
                        str(out)], cwd=checkout, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    for rank in range(2):
        rec = json.loads((out / f"rank{rank}.json").read_text())
        for key in ("models", "criterion", "pointnet2_modules"):
            path = Path(rec[key]).resolve()
            assert path.is_relative_to(PACKAGE.resolve()), f"rank {rank}: {key} from {path}"
        assert rec["nsync"] > 0
        assert rec["converted_keys"] == rec["plain_keys"]
