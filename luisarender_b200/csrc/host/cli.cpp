// luisa-render-cli — same command line as the reference's src/apps/cli.cpp:59-185:
//   luisa-render-cli -b <backend> [-d <index>] [-D key=value]... <scene file>
// Parses the scene (host library), uploads the flattened scene to the CUDA radiance library and renders
// every camera to its `file` (default <scene dir>/render.exr).  `-b cuda` selects the sm_90a backend; any
// other backend name is an error here (north_star: no multi-backend dispatch, no CPU fallback).
//
// Multi-GPU (SURVEY.md §8e; the reference is single-device): one PROCESS per GPU.  `--gpus N` makes this process a launcher
// that starts N copies of itself (RANK / WORLD_SIZE / LOCAL_RANK in the environment, as torchrun would set them — a torchrun
// or mpirun launch of the plain command works too) and waits for them.  Every rank parses the scene, renders the tiles it owns
// (lrk_balance_shards), and one lrk_reduce_film (NCCL) sums the raw films on rank 0, which writes the image.  The NCCL unique id
// travels through a file (LRK_COMM_ID_FILE, default /tmp/lrk_comm_<MASTER_PORT>.id): rank 0 writes it, the others wait for it.
//
// Adaptive sampling (an extension; the reference has none): `--adaptive <threshold>` renders with lrk_render_adaptive, from
// `--adaptive-min-spp` samples per pixel (default 16, at most the camera's spp) up to the camera's spp.
//
// Denoising (an extension): `--denoise` renders G-buffer films (lrk_set_option("gbuffer")) and also writes lrk_denoise's image to
// <stem>.denoised<ext> next to the camera's file, which is written as without it.  One GPU only: the G-buffer is not reduced.
//
// Light tree (an extension): `--light-tree` sets lrk_set_option("light_tree", 1) before the upload, so that next-event estimation
// picks its lights by power, distance and orientation.  Surface integrator only: a volume scene fails with the library's message.
//
// Solid-angle light sampling (an extension): `--light-solid-angle` sets lrk_set_option("light_solid_angle", 1) before the upload, so
// that next-event estimation samples the point on an emissive triangle uniformly in solid angle.  Surface integrator only, as above.
//
// Triangle-level light trees (an extension): `--light-tree-triangles` sets the options "light_tree" and "light_tree_triangles", so
// that the light tree also picks the emissive triangle by power, distance and orientation.  Surface integrator only, as above.
//
// Resampled light sampling (an extension): `--light-candidates <n>` sets lrk_set_option("light_candidates", n) before the upload;
// for n from 2 to 32, next-event estimation draws n candidates with the light sampling the flags above choose and traces the shadow
// ray of one, picked by its unshadowed contribution.  0 and 1 keep one light sample.  Surface integrator only, as above.
//
// Receiver-aware light sampling (an extension): `--light-receiver` sets lrk_set_option("light_receiver", 1) before the upload, so
// that the light tree and the solid-angle sampler also weigh by the shading point's normal.  With --light-tree, --light-tree-triangles
// or --light-solid-angle; alone, the upload fails with the library's message.  Surface integrator only, as above.
#include <sys/stat.h>
#include <sys/wait.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../../include/lrh.h"

namespace {

// the light-sampling flags: the options each sets to 1 before the upload
struct LightFlag {
    const char *flag, *help;
    std::vector<const char *> options;
};
const LightFlag kLightFlags[] = {
    {"--light-tree", "Pick next-event lights from a light tree (power, distance, orientation)", {"light_tree"}},
    {"--light-solid-angle", "Sample next-event light points uniformly in solid angle, not by area", {"light_solid_angle"}},
    {"--light-tree-triangles", "Also pick the emissive triangle from the light tree (implies --light-tree)", {"light_tree", "light_tree_triangles"}},
    {"--light-receiver", "Weigh tree lights and solid-angle points by the shading normal", {"light_receiver"}},
};

void usage() {
    std::printf("Usage:\n  luisa-render-cli [OPTION...] <file>\n\n"
                "  -b, --backend <backend>      Compute backend name (cuda)\n"
                "  -d, --device <index>         Compute device index (default: -1)\n"
                "      --scene <file>           Path to scene description file\n"
                "  -D, --define <key>=<value>   Parameter definitions to override scene description macros.\n"
                "      --gpus <n>               Render on n GPUs, one process each (tiles sharded, films summed on GPU 0)\n"
                "      --adaptive <threshold>   Adaptive sampling: stop 8x4 pixel blocks whose relative error is below threshold\n"
                "      --adaptive-min-spp <n>   Samples per pixel of the first adaptive round (default 16, at most the camera's spp)\n"
                "      --denoise                Also write the denoised image to <stem>.denoised<ext> (one GPU only)\n");
    for (const LightFlag &l : kLightFlags) std::printf("      %-25s%s\n", l.flag, l.help);
    std::printf("      --light-candidates <n>   Resample next-event lights from n candidates (2 to 32; 0 or 1: one light sample)\n");
    std::printf("  -h, --help                   Display this help message\n");
}

[[noreturn]] void die(const std::string &msg) {
    std::fprintf(stderr, "[error] %s\n", msg.c_str());
    std::abort();// the reference's LUISA_ERROR logs and aborts (logging.h:63,107)
}

uint32_t env_u32(const char *name, uint32_t fallback) {
    const char *v = std::getenv(name);
    return v != nullptr && *v != '\0' ? static_cast<uint32_t>(std::strtoul(v, nullptr, 10)) : fallback;
}

std::string comm_id_file() {
    if (const char *f = std::getenv("LRK_COMM_ID_FILE"); f != nullptr && *f != '\0') return f;
    const char *port = std::getenv("MASTER_PORT");
    return std::string("/tmp/lrk_comm_") + (port != nullptr ? port : "0") + ".id";
}

// rank 0 publishes the id (write + rename: never half a file), the others poll for it
void exchange_comm_id(uint32_t rank, uint8_t id[LRK_COMM_ID_BYTES]) {
    const std::string path = comm_id_file();
    if (rank == 0u) {
        if (lrk_comm_unique_id(id) != 0) die("NCCL is not available (libnccl.so.2): cannot render on several GPUs.");
        const std::string tmp = path + ".tmp";
        FILE *f = std::fopen(tmp.c_str(), "wb");
        if (f == nullptr || std::fwrite(id, 1, LRK_COMM_ID_BYTES, f) != LRK_COMM_ID_BYTES) die("Cannot write '" + tmp + "'.");
        std::fclose(f);
        if (std::rename(tmp.c_str(), path.c_str()) != 0) die("Cannot publish '" + path + "'.");
        return;
    }
    for (int attempt = 0; attempt < 6000; attempt++) {// up to 10 minutes: rank 0 may still be parsing a large scene
        struct stat st{};
        if (stat(path.c_str(), &st) == 0 && st.st_size == LRK_COMM_ID_BYTES) {
            FILE *f = std::fopen(path.c_str(), "rb");
            if (f != nullptr && std::fread(id, 1, LRK_COMM_ID_BYTES, f) == LRK_COMM_ID_BYTES) {
                std::fclose(f);
                return;
            }
            if (f != nullptr) std::fclose(f);
        }
        std::this_thread::sleep_for(std::chrono::milliseconds(100));
    }
    die("Timed out waiting for rank 0's communicator id in '" + path + "'.");
}

// --gpus N: start N copies of this command line, one per GPU
int launch_ranks(int gpus, int argc, char *argv[]) {
    std::string id_file = "/tmp/lrk_comm_" + std::to_string(getpid()) + ".id";
    std::remove(id_file.c_str());
    std::vector<pid_t> children;
    for (int r = 0; r < gpus; r++) {
        pid_t pid = fork();
        if (pid < 0) die("fork failed.");
        if (pid == 0) {
            setenv("RANK", std::to_string(r).c_str(), 1);
            setenv("LOCAL_RANK", std::to_string(r).c_str(), 1);
            setenv("WORLD_SIZE", std::to_string(gpus).c_str(), 1);
            setenv("LRK_COMM_ID_FILE", id_file.c_str(), 1);
            std::vector<char *> args;
            for (int i = 0; i < argc; i++) {
                std::string a{argv[i]};
                if (a == "--gpus") { i++; continue; }
                if (a.rfind("--gpus=", 0) == 0) continue;
                args.push_back(argv[i]);
            }
            args.push_back(nullptr);
            execv("/proc/self/exe", args.data());
            std::perror("execv");
            _exit(127);
        }
        children.push_back(pid);
    }
    int worst = 0;
    for (pid_t pid : children) {
        int status = 0;
        waitpid(pid, &status, 0);
        int code = WIFEXITED(status) ? WEXITSTATUS(status) : 128 + (WIFSIGNALED(status) ? WTERMSIG(status) : 0);
        if (code != 0 && worst == 0) worst = code;
    }
    std::remove(id_file.c_str());
    return worst;
}

// <dir>/<stem>.denoised<ext> for <dir>/<stem><ext>
std::string denoised_path(const std::string &file) {
    const size_t slash = file.find_last_of('/'), dot = file.find_last_of('.');
    if (dot == std::string::npos || (slash != std::string::npos && dot < slash)) return file + ".denoised";
    return file.substr(0, dot) + ".denoised" + file.substr(dot);
}

}// namespace

int main(int argc, char *argv[]) {
    std::string backend, scene_path;
    int device = -1, gpus = 1;
    bool denoise = false;
    std::vector<const char *> light_options;
    std::string adaptive_arg, min_spp_arg, candidates_arg;
    std::vector<std::string> keys, values;
    auto add_macro = [&](const std::string &d) {
        auto p = d.find('=');
        if (p == std::string::npos) {
            std::fprintf(stderr, "[warning] Invalid definition: %s\n", d.c_str());
            return;
        }
        auto k = d.substr(0, p), v = d.substr(p + 1);
        for (size_t i = 0; i < keys.size(); i++) {
            if (keys[i] == k) {
                std::fprintf(stderr, "[warning] Duplicate definition: %s = '%s'. Ignoring the previous one.\n", k.c_str(), v.c_str());
                values[i] = v;
                return;
            }
        }
        keys.push_back(k);
        values.push_back(v);
    };
    for (int i = 1; i < argc; i++) {
        std::string a{argv[i]};
        auto need = [&](const char *what) -> std::string {
            if (i + 1 >= argc) {
                std::fprintf(stderr, "[warning] Missing %s after %s.\n", what, a.c_str());
                usage();
                std::exit(-1);
            }
            return argv[++i];
        };
        if (a == "-h" || a == "--help") { usage(); return 0; }
        else if (a == "-b" || a == "--backend") backend = need("backend");
        else if (a.rfind("--backend=", 0) == 0) backend = a.substr(10);
        else if (a == "-d" || a == "--device") device = std::atoi(need("index").c_str());
        else if (a.rfind("--device=", 0) == 0) device = std::atoi(a.substr(9).c_str());
        else if (a == "--scene") scene_path = need("file");
        else if (a == "--gpus") gpus = std::atoi(need("count").c_str());
        else if (a.rfind("--gpus=", 0) == 0) gpus = std::atoi(a.substr(7).c_str());
        else if (a == "--adaptive") adaptive_arg = need("threshold");
        else if (a.rfind("--adaptive=", 0) == 0) adaptive_arg = a.substr(11);
        else if (a == "--adaptive-min-spp") min_spp_arg = need("count");
        else if (a.rfind("--adaptive-min-spp=", 0) == 0) min_spp_arg = a.substr(19);
        else if (a == "--denoise") denoise = true;
        else if (auto l = std::find_if(std::begin(kLightFlags), std::end(kLightFlags), [&](const LightFlag &f) { return a == f.flag; });
                 l != std::end(kLightFlags))
            light_options.insert(light_options.end(), l->options.begin(), l->options.end());
        else if (a == "--light-candidates") candidates_arg = need("count");
        else if (a.rfind("--light-candidates=", 0) == 0) candidates_arg = a.substr(19);
        else if (a == "-D" || a == "--define") add_macro(need("definition"));
        else if (a.rfind("-D", 0) == 0) add_macro(a.substr(2));
        else if (!a.empty() && a[0] == '-') std::fprintf(stderr, "[warning] Unrecognized options: %s\n", a.c_str());
        else scene_path = a;
    }
    if (scene_path.empty()) {
        std::fprintf(stderr, "[warning] Scene file not specified.\n");
        usage();
        return -1;
    }
    if (backend.empty()) {
        std::fprintf(stderr, "[warning] Failed to parse command line arguments: Option 'backend' has no value.\n");
        usage();
        return -1;
    }
    // the adaptive options are checked here, before the scene is read or a device is touched
    const bool adaptive = !adaptive_arg.empty();
    float threshold = 0.f;
    uint32_t min_spp = 16u;
    if (adaptive) {
        char *end = nullptr;
        threshold = std::strtof(adaptive_arg.c_str(), &end);
        if (end == adaptive_arg.c_str() || *end != '\0' || !std::isfinite(threshold) || threshold < 0.f) {
            std::fprintf(stderr, "[error] --adaptive takes a finite threshold >= 0, not '%s'.\n", adaptive_arg.c_str());
            return -1;
        }
    }
    if (!min_spp_arg.empty()) {
        char *end = nullptr;
        const unsigned long v = std::strtoul(min_spp_arg.c_str(), &end, 10);
        if (!adaptive || end == min_spp_arg.c_str() || *end != '\0' || min_spp_arg[0] == '-' || v < 2ul || v > 0xffffffffull) {
            std::fprintf(stderr, "[error] --adaptive-min-spp takes a count >= 2 and needs --adaptive, not '%s'.\n", min_spp_arg.c_str());
            return -1;
        }
        min_spp = static_cast<uint32_t>(v);
    }
    long candidates = -1;// -1: the option is left at its default
    if (!candidates_arg.empty()) {
        char *end = nullptr;
        candidates = std::strtol(candidates_arg.c_str(), &end, 10);
        if (end == candidates_arg.c_str() || *end != '\0' || candidates < 0 || candidates > 32) {
            std::fprintf(stderr, "[error] --light-candidates takes a count from 0 to 32, not '%s'.\n", candidates_arg.c_str());
            return -1;
        }
    }
    if (denoise && (gpus > 1 || env_u32("WORLD_SIZE", 1u) > 1u)) {
        std::fprintf(stderr, "[error] --denoise renders on one GPU: the G-buffer of sharded renders is not reduced.\n");
        return -1;
    }
    for (auto &c : backend) c = static_cast<char>(std::tolower(static_cast<unsigned char>(c)));
    if (backend != "cuda") die("Backend '" + backend + "' is not available: this build ships the sm_90a CUDA backend only (-b cuda).");
    if (gpus > 1) return launch_ranks(gpus, argc, argv);
    const uint32_t rank = env_u32("RANK", 0u), world = std::max(1u, env_u32("WORLD_SIZE", 1u));
    if (rank >= world) die("RANK must be below WORLD_SIZE.");
    if (world > 1u && device < 0) device = static_cast<int>(env_u32("LOCAL_RANK", rank));
    const bool root = rank == 0u;

    std::vector<const char *> k, v;
    for (size_t i = 0; i < keys.size(); i++) {
        std::printf("[info] Found CLI Macro: %s = %s\n", keys[i].c_str(), values[i].c_str());
        k.push_back(keys[i].c_str());
        v.push_back(values[i].c_str());
    }
    auto t0 = std::chrono::steady_clock::now();
    lrh_scene *scene = nullptr;
    if (lrh_scene_load(scene_path.c_str(), k.data(), v.data(), static_cast<uint32_t>(k.size()), &scene) != 0) die(lrh_last_error());
    auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    lrh_scene_info info{};
    lrh_scene_get_info(scene, &info);
    std::printf("[info] Parsed and flattened scene '%s' in %.1f ms (BVH build %.1f ms).\n", scene_path.c_str(),
                ms(t0, std::chrono::steady_clock::now()), info.bvh_build_ms);
    std::printf("[info] Geometry built with %llu triangles (%llu unique, %u meshes, %u instances).\n",
                static_cast<unsigned long long>(info.instanced_triangles), static_cast<unsigned long long>(info.unique_triangles),
                info.meshes, info.instances);

    lrk_device_cfg cfg{};
    cfg.device_index = device;
    lrk_ctx *ctx = nullptr;
    if (int rc = lrk_create(&cfg, &ctx); rc != 0) die("Failed to create the CUDA device context (lrk_create = " + std::to_string(rc) + ").");
    if (denoise && lrk_set_option(ctx, "gbuffer", 1) != 0) die(lrk_last_error(ctx));
    for (const char *option : light_options)
        if (lrk_set_option(ctx, option, 1) != 0) die(lrk_last_error(ctx));
    if (candidates >= 0 && lrk_set_option(ctx, "light_candidates", candidates) != 0) die(lrk_last_error(ctx));
    if (world > 1u) {
        uint8_t id[LRK_COMM_ID_BYTES];
        exchange_comm_id(rank, id);
        if (lrk_comm_init(ctx, id, rank, world) != 0) die(lrk_last_error(ctx));
        std::printf("[info] Rank %u of %u on device %d.\n", rank, world, device);
    }
    for (uint32_t cam = 0; cam < info.cameras; cam++) {
        lrk_scene_desc desc{};
        if (lrh_scene_get_desc(scene, cam, &desc) != 0) die(lrh_last_error());
        if (lrk_upload_scene(ctx, &desc) != 0) {
            std::string msg = lrk_last_error(ctx);
            if (msg.find("No lights in scene") != std::string::npos) {// reference: warn and skip (wave_path.cpp:224-228)
                std::fprintf(stderr, "[warning] %s\n", msg.c_str());
                continue;
            }
            die(msg);
        }
        // N ranks: each takes its share of a cost-balanced tile assignment (a one-sample probe of the frame on every rank, no
        // communication); the volume integrator has no probe and takes the static tile map
        if (world > 1u && lrk_balance_shards(ctx, rank, world, 32u, 1u) != 0 && lrk_set_shard(ctx, rank, world, 32u) != 0) die(lrk_last_error(ctx));
        const uint32_t w = desc.camera.resolution[0], h = desc.camera.resolution[1], spp = desc.camera.spp;
        std::printf("[info] Wavefront path tracing configurations: resolution = %ux%u, spp = %u.\n", w, h, spp);
        std::printf("[info] Rendering started.\n");
        const lrk_adaptive ap{std::min(min_spp, spp), spp, threshold, 0u};
        if (adaptive ? lrk_render_adaptive(ctx, &ap) != 0 : lrk_render(ctx, 0u, spp) != 0) die(lrk_last_error(ctx));
        if (world > 1u && lrk_reduce_film(ctx, 0u) != 0) die(lrk_last_error(ctx));
        lrk_stats st{};
        lrk_get_stats(ctx, &st);
        if (adaptive) {// this rank's pixels: samples against a uniform render, and the rounds it took (counts are min_spp * 2^k or spp)
            std::vector<uint32_t> counts(static_cast<size_t>(w) * h);
            if (lrk_download_sample_counts(ctx, counts.data()) != 0) die(lrk_last_error(ctx));
            uint64_t owned = 0u;
            uint32_t top = 0u;
            for (uint32_t c : counts) {
                owned += c != 0u ? 1u : 0u;
                top = std::max(top, c);
            }
            uint32_t rounds = 1u;
            for (uint32_t level = ap.min_spp; level < top; level = static_cast<uint32_t>(std::min<uint64_t>(2ull * level, spp))) rounds++;
            const std::string who = world > 1u ? "Rank " + std::to_string(rank) + ": a" : "A";
            std::printf("[info] %sdaptive sampling (threshold %g, %u to %u spp): %llu samples, %.2f %% of a uniform render, %u rounds.\n", who.c_str(),
                        static_cast<double>(threshold), ap.min_spp, spp, static_cast<unsigned long long>(st.samples),
                        owned != 0u ? 100.0 * static_cast<double>(st.samples) / (static_cast<double>(owned) * spp) : 0.0, rounds);
        }
        if (world > 1u) std::printf("[info] Rank %u rendered its tiles in %.3f ms (film reduce %.3f ms).\n", rank, st.render_ms, st.reduce_ms);
        if (!root) continue;
        std::printf("[info] Rendering finished in %.3f ms.\n", st.render_ms + st.reduce_ms);
        std::printf("[info] %.2f Msamples/s, %.2f Mrays/s (%llu closest + %llu shadow rays).\n",
                    static_cast<double>(st.samples) / st.render_ms * 1e-3,
                    static_cast<double>(st.closest_rays + st.shadow_rays) / st.render_ms * 1e-3,
                    static_cast<unsigned long long>(st.closest_rays), static_cast<unsigned long long>(st.shadow_rays));
        std::vector<float> pixels(static_cast<size_t>(w) * h * 4u);
        if (lrk_download_film(ctx, pixels.data()) != 0) die(lrk_last_error(ctx));
        const char *file = lrh_scene_camera_file(scene, cam);
        if (lrh_save_image(file, pixels.data(), w, h) != 0) std::fprintf(stderr, "[warning] %s\n", lrh_last_error());
        else std::printf("[info] Saved film to '%s'.\n", file);
        if (denoise) {
            if (lrk_denoise(ctx, pixels.data()) != 0) die(lrk_last_error(ctx));
            const std::string out = denoised_path(file);
            if (lrh_save_image(out.c_str(), pixels.data(), w, h) != 0) std::fprintf(stderr, "[warning] %s\n", lrh_last_error());
            else std::printf("[info] Saved denoised film to '%s'.\n", out.c_str());
        }
    }
    lrk_destroy(ctx);
    lrh_scene_destroy(scene);
    return 0;
}
