"""Import-path shim: keeps the reference dotted `_target_` paths (configs/*.yaml) resolving to the H100 engine (seed-x_b200/)."""
