// mtsb200 -- stand-alone driver over the C-ABI with the reference CLI's contract for this path
// (src/mitsuba/mitsuba.cpp:129-417: `mitsuba [-o out] [-D key=value]... scene.xml`).  Writes a PFM (linear RGB float).
#include "../../include/b2mts.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

static void usage() {
    fprintf(stderr, "usage: mtsb200 [-o out.pfm] [-D key=value]... [-g gpu] [-q] [--accel-build host|device] scene.xml\n"
                    "  renders <scene.xml> with the GPU wavefront `path` integrator (no CPU fallback)\n"
                    "  --accel-build  builder of the acceleration structure: host (multi-threaded CPU, the default) or device (GPU)\n");
}

int main(int argc, char **argv) {
    std::string out, scene;
    std::vector<const char *> defs;
    int gpu = 0;
    bool quiet = false;
    int accelBuild = B2_ACCEL_BUILD_HOST;
    for (int i = 1; i < argc; ++i) {
        if (!strcmp(argv[i], "-o") && i + 1 < argc) out = argv[++i];
        else if (!strcmp(argv[i], "-D") && i + 1 < argc) defs.push_back(argv[++i]);
        else if (!strncmp(argv[i], "-D", 2) && argv[i][2]) defs.push_back(argv[i] + 2);
        else if (!strcmp(argv[i], "-g") && i + 1 < argc) gpu = atoi(argv[++i]);
        else if (!strcmp(argv[i], "-q")) quiet = true;
        else if (!strcmp(argv[i], "--accel-build") && i + 1 < argc) {
            const char *m = argv[++i];
            if (!strcmp(m, "host")) accelBuild = B2_ACCEL_BUILD_HOST;
            else if (!strcmp(m, "device")) accelBuild = B2_ACCEL_BUILD_DEVICE;
            else { fprintf(stderr, "--accel-build must be host or device, not %s\n", m); usage(); return 2; }
        }
        else if (!strcmp(argv[i], "-h")) { usage(); return 0; }
        else if (argv[i][0] == '-') { fprintf(stderr, "unknown option %s\n", argv[i]); usage(); return 2; }
        else scene = argv[i];
    }
    if (scene.empty()) { usage(); return 2; }
    if (out.empty()) { out = scene; size_t k = out.rfind('.'); if (k != std::string::npos) out.resize(k); out += ".pfm"; } // mitsuba.cpp:381-386
    b2_ctx *ctx = nullptr;
    if (b2_context_create(gpu, &ctx)) { fprintf(stderr, "error: %s\n", b2_last_error(nullptr)); return 1; }
    if (b2_context_set_accel_build(ctx, accelBuild)) { fprintf(stderr, "error: %s\n", b2_last_error(ctx)); return 1; }
    b2_scene *sc = nullptr;
    b2_render_params rp;
    if (b2_load_xml(ctx, scene.c_str(), defs.data(), (int) defs.size(), &sc, &rp)) { fprintf(stderr, "error: %s\n", b2_last_error(ctx)); return 1; }
    int W = 0, H = 0;
    b2_scene_film_size(sc, &W, &H);
    std::vector<float> film((size_t) W * H * 5), rgb((size_t) W * H * 3);
    if (b2_render(sc, &rp, film.data())) { fprintf(stderr, "error: %s\n", b2_last_error(ctx)); return 1; }
    b2_film_develop(film.data(), W, H, rgb.data());
    b2_stats st;
    b2_get_stats(sc, &st);
    FILE *f = fopen(out.c_str(), "wb");
    if (!f) { fprintf(stderr, "cannot write %s\n", out.c_str()); return 1; }
    fprintf(f, "PF\n%d %d\n-1.0\n", W, H);
    for (int y = H - 1; y >= 0; --y) fwrite(&rgb[(size_t) y * W * 3], sizeof(float), (size_t) W * 3, f); // PFM is bottom-up
    fclose(f);
    if (!quiet)
        printf("Render time: %.3f s  (%.1f Msamples/s, %llu samples, avg path length %.3f, %llu rays, %llu shadow rays) -> %s\n", st.ms_total / 1e3,
               st.samples / (st.ms_total * 1e3), (unsigned long long) st.samples, (double) st.path_length_sum / (double) st.samples,
               (unsigned long long) st.rays, (unsigned long long) st.shadow_rays, out.c_str());
    b2_scene_destroy(sc);
    b2_context_destroy(ctx);
    return 0;
}
