// build.rs of the crate that binds liblurk_b200 (C ABI: include/lurk_b200.h of the lurk-beta_b200 repository).
// The library is a plain shared object built by `python -c "import __graft_entry__ as g; g.build()"` (nvcc, sm_90a);
// point LURK_B200_LIB_DIR at the directory that holds liblurk_b200.so.
use std::env;

fn main() {
    println!("cargo:rerun-if-env-changed=LURK_B200_LIB_DIR");
    if let Ok(dir) = env::var("LURK_B200_LIB_DIR") {
        println!("cargo:rustc-link-search=native={dir}");
        println!("cargo:rustc-link-arg=-Wl,-rpath,{dir}");
    }
    println!("cargo:rustc-link-lib=dylib=lurk_b200");
}
