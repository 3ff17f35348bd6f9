// main.cpp -- drop-in command line of waifu2x-converter-cpp (reference src/main.cpp) on top of the GPU hot path.
// Same flags, defaults, progress messages, output naming and exit codes; the two convertWithModels calls
// (src/main.cpp:96,148) go to libw2x_b200.so through host/w2xc.hpp, everything around them is restated from
// src/main.cpp line by line with host/imgproc.hpp + host/imageio.hpp standing in for OpenCV.
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "imageio.hpp"
#include "imgproc.hpp"
#include "w2xc.hpp"

namespace {

// ---- a TCLAP-shaped parser: ValueArg flags only, ' ' delimiter, --help / --version / -- (reference src/main.cpp:26-71) ----
struct Arg {
    std::string flag, name, desc, type;
    bool required;
    std::string def;
    std::vector<std::string> allowed;
    std::string value;
    bool set = false;
    bool hidden = false;   // accepted, but not part of the reference's flag surface: left out of --help and the usage lines
};

struct CmdLine {
    std::string prog, message = "waifu2x reimplementation using OpenCV", version = "1.0.0";
    std::vector<Arg> args;

    Arg &add(const char *flag, const char *name, const char *desc, bool req, const char *def, const char *type,
             std::vector<std::string> allowed = {}) {
        Arg a; a.flag = flag; a.name = name; a.desc = desc; a.required = req; a.def = def; a.type = type; a.allowed = allowed; a.value = def;
        args.push_back(a);
        return args.back();
    }
    std::string id(const Arg &a) const { return (a.flag.empty() ? "" : "-" + a.flag + " ") + "(--" + a.name + ")"; }
    std::string shortid(const Arg &a) const {
        std::string t = a.allowed.empty() ? a.type : "";
        for (size_t i = 0; i < a.allowed.size(); i++) t += (i ? "|" : "") + a.allowed[i];
        std::string s = (a.flag.empty() ? "--" + a.name : "-" + a.flag) + " <" + t + ">";
        return a.required ? s : "[" + s + "]";
    }
    void brief(std::ostream &os) const {
        os << "Brief USAGE: \n   " << prog << " ";
        for (auto it = args.rbegin(); it != args.rend(); ++it)
            if (!it->hidden) os << " " << shortid(*it);
        os << " [--] [--version] [-h]\n\nFor complete USAGE and HELP type: \n   " << prog << " --help\n\n";
    }
    [[noreturn]] void parse_error(const std::string &argid, const std::string &text) const {
        std::cerr << "PARSE ERROR: " << argid << "\n             " << text << "\n\n";
        brief(std::cerr);
        std::exit(1);   // TCLAP StdOutput::failure -> exit(1)
    }
    void usage() const {
        std::cout << "\nUSAGE: \n\n   " << prog << " ";
        for (auto it = args.rbegin(); it != args.rend(); ++it)
            if (!it->hidden) std::cout << " " << shortid(*it);
        std::cout << " [--] [--version] [-h]\n\n\nWhere: \n\n";
        for (auto it = args.rbegin(); it != args.rend(); ++it) {
            if (it->hidden) continue;
            std::string t = it->allowed.empty() ? it->type : "";
            for (size_t i = 0; i < it->allowed.size(); i++) t += (i ? "|" : "") + it->allowed[i];
            std::cout << "   " << (it->flag.empty() ? "" : "-" + it->flag + " <" + t + ">,  ") << "--" << it->name << " <" << t << ">\n     "
                      << (it->required ? "(required)  " : "") << it->desc << "\n\n";
        }
        std::cout << "   --,  --ignore_rest\n     Ignores the rest of the labeled arguments following this flag.\n\n"
                     "   --version\n     Displays version information and exits.\n\n"
                     "   -h,  --help\n     Displays usage information and exits.\n\n\n   " << message << "\n\n";
    }
    void parse(int argc, char **argv) {
        prog = argv[0];
        size_t slash = prog.find_last_of('/');
        if (slash != std::string::npos) prog = prog.substr(slash + 1);
        for (int i = 1; i < argc; i++) {
            std::string tok = argv[i];
            if (tok == "--" || tok == "--ignore_rest") break;
            if (tok == "-h" || tok == "--help") { usage(); std::exit(0); }
            if (tok == "--version") { std::cout << "\n" << prog << "  version: " << version << "\n\n"; std::exit(0); }
            Arg *hit = nullptr;
            for (auto &a : args)
                if ((tok.rfind("--", 0) == 0 && tok.substr(2) == a.name) || (!a.flag.empty() && tok == "-" + a.flag)) hit = &a;
            if (!hit) parse_error("Argument: " + tok, "Couldn't find match for argument");
            if (hit->set) parse_error("Argument: " + id(*hit), "Argument already set!");
            if (i + 1 >= argc) parse_error("Argument: " + id(*hit), "Missing a value for this argument!");
            hit->value = argv[++i];
            hit->set = true;
            if (hit->type == "integer" || hit->type == "double") {
                char *end = nullptr;
                if (hit->type == "integer") std::strtol(hit->value.c_str(), &end, 10); else std::strtod(hit->value.c_str(), &end);
                if (end == hit->value.c_str() || *end) parse_error("Argument: " + id(*hit), "Couldn't read argument value from string '" + hit->value + "'");
            }
            if (!hit->allowed.empty()) {
                bool ok = false;
                for (auto &v : hit->allowed) ok = ok || v == hit->value;
                if (!ok) {
                    std::string c;
                    for (size_t k = 0; k < hit->allowed.size(); k++) c += (k ? "|" : "") + hit->allowed[k];
                    parse_error("Argument: " + id(*hit), "Value '" + hit->value + "' does not meet constraint: " + c);
                }
            }
        }
        for (auto &a : args)
            if (a.required && !a.set) parse_error(" ", "Required argument missing: " + a.name);   // TCLAP: CmdLineParseException with argId " "
    }
    const std::string &get(const char *name) const {
        for (auto &a : args) if (a.name == name) return a.value;
        static std::string empty;
        return empty;
    }
};

w2xc::Plane plane_of(const w2ximg::Image3f &im, int c) {              // cv::split, one channel
    w2xc::Plane p(im.width, im.height);
    w2ximg::get_channel(im, c, p.data, p.stride_bytes / 4);
    return p;
}
// channel c of cv::resize(im, Size(dw, dh), 0, 0, INTER_NEAREST) (src/main.cpp:135-139: resize, then split, then only [0] is used)
w2xc::Plane plane_of_nearest(const w2ximg::Image3f &im, int c, int dw, int dh) {
    w2xc::Plane p(dw, dh);
    w2ximg::resize_nearest_channel(im, c, dw, dh, p.data, p.stride_bytes / 4);
    return p;
}

}  // namespace

int main(int argc, char **argv) {
    CmdLine cmd;
    cmd.add("i", "input_file", "path to input image file (you should input full path)", true, "", "string");
    cmd.add("o", "output_file", "path to output image file (you should input full path)", false, "(auto)", "string");
    cmd.add("m", "mode", "image processing mode", false, "noise_scale", "string", {"noise", "scale", "noise_scale"});
    cmd.add("", "noise_level", "noise reduction level", false, "1", "integer", {"1", "2"});
    cmd.add("", "scale_ratio", "custom scale ratio", false, "2.0", "double");
    cmd.add("", "model_dir", "path to custom model directory (don't append last / )", false, "models", "string");
    cmd.add("j", "jobs", "number of threads launching at the same time", false, "4", "integer");
    // the sibling of -j for this implementation (src/main.cpp:58-60 is where the reference declares -j): planes are cut into
    // this many row bands, one per GPU, halo rows exchanged between the GPUs after every layer; W2X_GPUS does the same
    cmd.add("", "gpus", "number of GPUs the conversion is spread over", false, "1", "integer").hidden = true;
    // test-time augmentation (the -tta / --tta switch of later waifu2x front ends): every pass is the mean of its conversions of the
    // Y plane's 8 flips and transposes, at 8x the GPU work; stdout and output naming stay as without it
    cmd.add("", "tta", "average every pass over the 8 flips and transposes of the plane", false, "0", "integer", {"0", "1"}).hidden = true;
    cmd.parse(argc, argv);
    const bool tta = cmd.get("tta") == "1";
    {
        const int gpus = w2xc::gpuRuntime::plannedNumberOfGpus(std::atoi(cmd.get("gpus").c_str()));
        if (tta && gpus > 1) {   // a TTA step has no multi-GPU form (w2x_multi_convert_chain refuses it)
            std::cerr << "Error : --tta 1 runs on one GPU; it cannot be combined with " << gpus << " GPUs (--gpus / W2X_GPUS / W2X_DEVICES)." << std::endl;
            std::exit(1);
        }
    }
    if (std::atoi(cmd.get("gpus").c_str()) > 1) w2xc::gpuRuntime::setNumberOfGpus(std::atoi(cmd.get("gpus").c_str()));
    // CUDA context creation (~0.2 s) overlaps image decoding, colour conversion and model parsing; joined before the first conversion
    std::thread gpu_warmup([] { w2xc::gpuRuntime::warmup(); });
    // every way out of main below joins it first: std::exit runs the static destructors, and the runtime must not still be under construction
    auto leave = [&](int code) {
        if (gpu_warmup.joinable()) gpu_warmup.join();
        std::exit(code);
    };
    const bool timing = std::getenv("W2X_CLI_TIMING") != nullptr;   // stage times (ms) as one JSON line on stderr
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_start = now();
    double t_conv = 0.0, t_ctx_wait = 0.0;
    auto wait_for_gpu = [&] {                      // the part of the CUDA context creation the host work before it did not hide
        const double t0 = now();
        if (gpu_warmup.joinable()) gpu_warmup.join();
        t_ctx_wait += now() - t0;
    };

    const std::string mode = cmd.get("mode"), inputFile = cmd.get("input_file"), modelDir = cmd.get("model_dir");
    const int nrLevel = std::atoi(cmd.get("noise_level").c_str());
    // the model files this run will ask for are read and parsed in the background while the image is decoded (silently: failures are
    // reported where the reference reports them, by the generateModelFromJSON calls below)
    if (mode == "noise" || mode == "noise_scale") w2xc::modelUtility::prefetchModelFromJSON(modelDir + "/noise" + std::to_string(nrLevel) + "_model.json");
    if (mode == "scale" || mode == "noise_scale") w2xc::modelUtility::prefetchModelFromJSON(modelDir + "/scale2.0x_model.json");
    const double scaleRatio = std::strtod(cmd.get("scale_ratio").c_str(), nullptr);

    // load image file (src/main.cpp:74-76)
    std::string ioerr;
    w2xio::Image8 in8 = w2xio::imread(inputFile, &ioerr);
    if (in8.empty()) {
        std::cerr << "Error : couldn't read image " << inputFile << " (" << ioerr << ")" << std::endl;
        leave(-1);
    }
    const double t_read = now();
    w2ximg::Image3f image = w2ximg::from_u8(in8.bgr.data(), in8.width, in8.height);
    w2ximg::rgb2yuv(image);

    w2xc::modelUtility::getInstance().setNumberOfJobs(std::atoi(cmd.get("jobs").c_str()));   // :79
    // (-j bounds the reference's filter threads; here it bounds the host image plumbing's row workers, the GPU does the filtering)

    const bool noisePhase = mode == "noise" || mode == "noise_scale", scalePhase = mode == "scale" || mode == "noise_scale";
    const int iterTimesTwiceScaling = static_cast<int>(std::ceil(std::log2(scaleRatio)));   // :107-108
    std::vector<std::unique_ptr<w2xc::Model>> noiseModels, scaleModels;
    if (noisePhase && !w2xc::modelUtility::generateModelFromJSON(modelDir + "/noise" + std::to_string(nrLevel) + "_model.json", noiseModels))
        leave(-1);                                                                          // :88-89
    // The Y plane after each pass depends only on the Y plane before it (split / merge / an exact 2x nearest resize copy values, the
    // bicubic Y channel is overwritten at :148-154, U and V never feed back into Y).  So the noise pass and every 2x iteration run as
    // ONE chain that keeps Y on the device (with --gpus n > 1: its row bands, each on its GPU), while the bicubic iterations of U and
    // V run here on the host.  -m noise, no usable device and a scale model that does not load keep the per-pass path below.
    // With --tta 1 every pass is a TTA step of the chain (-m noise a one-step chain); without a device the chain call reports it.
    bool chained = false;                          // the 2x iterations run in the chain
    if (scalePhase && iterTimesTwiceScaling >= 1 && w2xc::modelUtility::tryGenerateModelFromJSON(modelDir + "/scale2.0x_model.json", scaleModels)) {
        wait_for_gpu();
        chained = tta || w2xc::gpuRuntime::context() != nullptr;
    }
    const bool noiseChained = noisePhase && (chained || tta);
    if (chained || noiseChained) {
        struct Progress {
            bool noise;
            int failedStep = -1;
            static void step(int k, void *user) {                                           // stdout keeps the reference's line order
                Progress *p = static_cast<Progress *>(user);
                p->failedStep = k;
                const int it = p->noise ? k : k + 1;                                        // 2x iteration number, 0 = the noise pass
                if (it == 1) std::cout << "start scaling" << std::endl;                     // :123
                if (it >= 1) std::cout << "#" << std::to_string(it) << " 2x scaling..." << std::endl;   // :129-130
            }
        } progress{noisePhase};
        std::vector<w2xc::ChainStep> steps;
        if (noisePhase) steps.push_back({&noiseModels, false, tta});
        const int chainedIterations = chained ? iterTimesTwiceScaling : 0;
        for (int i = 0; i < chainedIterations; i++) steps.push_back({&scaleModels, true, tta});
        w2xc::Plane imageY = plane_of(image, 0), out;
        wait_for_gpu();
        // the bicubic iterations (:144) of U and V: w2ximg::resize computes every channel from that channel alone, so U and V do not
        // depend on the Y values they are resized along with
        std::thread colour([&] {
            for (int i = 0; i < chainedIterations; i++) image = w2ximg::resize(image, image.width * 2, image.height * 2, w2ximg::CUBIC);
        });
        const double t0 = now();
        const bool ok = w2xc::convertChainWithModels(imageY, out, steps, &Progress::step, &progress);
        t_conv += now() - t0;
        colour.join();
        if (!ok) {
            if (noisePhase && progress.failedStep <= 0) leave(-1);                          // the noise pass failed (see below)
            std::cerr << "w2xc::convertWithModels : something error has occured.\nstop." << std::endl;
            leave(1);
        }
        w2ximg::set_channel(image, 0, out.data, out.stride_bytes / 4);                    // merge, :98 and :154
    }

    // ===== Noise Reduction Phase ===== (:82-100)
    if (noisePhase && !noiseChained) {
        std::vector<std::unique_ptr<w2xc::Model>> &models = noiseModels;
        w2xc::Plane imageY = plane_of(image, 0), out;
        wait_for_gpu();
        const double t0 = now();
        // The reference ignores the return value here (:96) because a failing layer has already ended the process inside
        // convertWithModelsBasic (src/convertRoutine.cpp:69: std::exit(-1)).  The library never exits, so the same outcome
        // is produced here: no device, out of memory or a CUDA error must not write the un-denoised image with exit code 0.
        if (!w2xc::convertWithModels(imageY, out, models) || out.empty()) leave(-1);
        t_conv += now() - t0;
        w2ximg::set_channel(image, 0, out.data, out.stride_bytes / 4);
    }

    // ===== scaling phase ===== (:104-169)
    if (scalePhase) {
        double shrinkRatio = 0.0;
        if (static_cast<int>(scaleRatio) != std::pow(2, iterTimesTwiceScaling))
            shrinkRatio = scaleRatio / std::pow(2.0, static_cast<double>(iterTimesTwiceScaling));
        std::vector<std::unique_ptr<w2xc::Model>> &models = scaleModels;
        // :120-121 (when the quiet load above failed, this one fails again and reports it here, after the noise pass, as the reference does)
        if (models.empty() && !w2xc::modelUtility::generateModelFromJSON(modelDir + "/scale2.0x_model.json", models)) leave(-1);
        if (!chained) std::cout << "start scaling" << std::endl;
        for (int nIteration = 0; nIteration < iterTimesTwiceScaling && !chained; nIteration++) {
            std::cout << "#" << std::to_string(nIteration + 1) << " 2x scaling..." << std::endl;
            const int w2 = image.width * 2, h2 = image.height * 2;
            w2xc::Plane imageY = plane_of_nearest(image, 0, w2, h2), out;                 // :135-139 (only the Y plane of the nearest image is used)
            w2ximg::Image3f bicubic = w2ximg::resize(image, w2, h2, w2ximg::CUBIC);      // :144
            wait_for_gpu();
            const double t0 = now();
            if (!w2xc::convertWithModels(imageY, out, models)) {
                std::cerr << "w2xc::convertWithModels : something error has occured.\nstop." << std::endl;
                leave(1);
            }
            t_conv += now() - t0;
            w2ximg::set_channel(bicubic, 0, out.data, out.stride_bytes / 4);              // merge, :154
            image = std::move(bicubic);
        }
        if (shrinkRatio != 0.0) {                                                           // :158-167
            int lw = static_cast<int>(static_cast<double>(image.width * shrinkRatio));
            int lh = static_cast<int>(static_cast<double>(image.height * shrinkRatio));
            image = w2ximg::resize(image, lw, lh, w2ximg::LINEAR);
        }
    }

    w2ximg::yuv2rgb(image);                                                                 // :171
    std::vector<uint8_t> out8 = w2ximg::to_u8(image);                                       // :172
    std::string outputFileName = cmd.get("output_file");
    if (outputFileName == "(auto)") {                                                       // :173-189
        outputFileName = inputFile;
        size_t tailDot = outputFileName.find_last_of('.');
        if (tailDot != std::string::npos) outputFileName.erase(tailDot, outputFileName.length());
        outputFileName = outputFileName + "(" + mode + ")";
        if (mode.find("noise") != mode.npos) outputFileName = outputFileName + "(Level" + std::to_string(nrLevel) + ")";
        if (mode.find("scale") != mode.npos) outputFileName = outputFileName + "(x" + std::to_string(scaleRatio) + ")";
        outputFileName += ".png";
    }
    const double t_write0 = now();
    if (!w2xio::imwrite(outputFileName, out8.data(), image.width, image.height)) {
        std::cerr << "Error : couldn't write " << outputFileName << std::endl;
        leave(-1);
    }
    if (timing)
        std::cerr << "{\"w2x_cli_timing_ms\": {\"imread\": " << t_read - t_start << ", \"convertWithModels\": " << t_conv
                  << ", \"cuda_context_wait\": " << t_ctx_wait << ", \"colour_resize_plumbing\": " << (t_write0 - t_read) - t_conv - t_ctx_wait
                  << ", \"imwrite\": " << now() - t_write0
                  << ", \"total\": " << now() - t_start << "}}" << std::endl;
    std::cout << "process successfully done!" << std::endl;
    if (gpu_warmup.joinable()) gpu_warmup.join();
    if (!std::getenv("W2X_CLI_FULL_TEARDOWN")) {   // the file is written and closed: skip the CUDA context / page-locked memory teardown (~0.1 s)
        std::cout.flush();
        std::cerr.flush();
        std::_Exit(0);
    }
    return 0;
}
