"""Drop-in counterparts of the reference's hot-path classes (same names, constructor kwargs, call
signatures and state-dict keys), executing on the sm_90a kernels.  Re-exported under the reference's
own dotted paths by the `model_lib/` tree at the repo root."""
