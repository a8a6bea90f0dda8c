//! The reference's renderer-agnostic image suite (test-renderers) against the H100 path: the third target next to
//! test-renderers/tests/ray-render.rs:6-19 and wgpu-render.rs.  The `-ray` / `-all` expectations apply: same
//! algorithm, same pixels (RendererId::Raytracer).

use clap::Parser as _;

use all_is_cubes_b200::B200Factory;
use all_is_cubes_render::camera::StandardCameras;
use all_is_cubes_render::HeadlessRenderer;
use test_renderers_types::{RendererFactory, RendererId, SuiteId};

#[derive(Clone, Debug)]
struct Factory(B200Factory);

impl RendererFactory for Factory {
    fn renderer_from_cameras(&self, cameras: StandardCameras) -> Box<dyn HeadlessRenderer + Send> {
        self.0.renderer_from_cameras(cameras)
    }
    fn id(&self) -> RendererId {
        RendererId::Raytracer
    }
    fn info(&self) -> String {
        self.0.info()
    }
}

#[tokio::main]
async fn main() -> test_renderers_runner::HarnessResult {
    let args = test_renderers_runner::HarnessArgs::parse();
    test_renderers_runner::initialize_logging(&args);
    let factory = Factory(B200Factory::new().expect("no H100 (sm_90) GPU: libaicb200 has no CPU fallback"));
    test_renderers_runner::harness_main(
        &args,
        RendererId::Raytracer,
        SuiteId::Renderers,
        test_renderers_cases::all_tests,
        move |_label| std::future::ready(factory.clone()),
        None,
    )
    .await
}
