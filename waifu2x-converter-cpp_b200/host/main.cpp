// main.cpp -- drop-in command line of waifu2x-converter-cpp (reference src/main.cpp) on top of the GPU hot path.
// Same flags, defaults, progress messages, output naming and exit codes; the two convertWithModels calls
// (src/main.cpp:96,148) go to libw2x_b200.so through host/w2xc.hpp, everything around them is restated from
// src/main.cpp line by line with host/imgproc.hpp + host/imageio.hpp standing in for OpenCV.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <deque>
#include <filesystem>
#include <fstream>
#include <functional>
#include <iostream>
#include <map>
#include <memory>
#include <mutex>
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
    std::string alternative;   // a flag that may stand in for this required one; giving both is an error (TCLAP's xorAdd)
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
            for (auto &a : args)
                if (a.set && (a.alternative == hit->name || hit->alternative == a.name))
                    parse_error("Argument: " + id(*hit), "Mutually exclusive argument already set!");
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
            if (a.required && !a.set && (a.alternative.empty() || !isSet(a.alternative.c_str())))
                parse_error(" ", "Required argument missing: " + a.name);   // TCLAP: CmdLineParseException with argId " "
    }
    const std::string &get(const char *name) const {
        for (auto &a : args) if (a.name == name) return a.value;
        static std::string empty;
        return empty;
    }
    bool isSet(const char *name) const {
        for (auto &a : args) if (a.name == name) return a.set;
        return false;
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

// ---- the per-image host stages, shared by the single-image and the --input_list runs ----
// load image file (src/main.cpp:74); the message and false when it cannot be read
bool readImage(const std::string &inputFile, w2xio::Image8 &in8) {
    std::string ioerr;
    in8 = w2xio::imread(inputFile, &ioerr);
    if (!in8.empty()) return true;
    std::cerr << ("Error : couldn't read image " + inputFile + " (" + ioerr + ")\n") << std::flush;   // one write: batch workers share stderr
    return false;
}
w2ximg::Image3f yuvImage(const w2xio::Image8 &in8) {                    // :75-76
    w2ximg::Image3f image = w2ximg::from_u8(in8.bgr.data(), in8.width, in8.height);
    w2ximg::rgb2yuv(image);
    return image;
}
// the Y plane's passes as one chain (see main): the noise pass, then `iterations` 2x steps
std::vector<w2xc::ChainStep> chainSteps(bool noise, int iterations, bool tta, std::vector<std::unique_ptr<w2xc::Model>> &noiseModels,
                                        std::vector<std::unique_ptr<w2xc::Model>> &scaleModels) {
    std::vector<w2xc::ChainStep> steps;
    if (noise) steps.push_back({&noiseModels, false, tta});
    for (int i = 0; i < iterations; i++) steps.push_back({&scaleModels, true, tta});
    return steps;
}
// the bicubic iterations (:144) of U and V: w2ximg::resize computes every channel from that channel alone, so U and V do not depend
// on the Y values they are resized along with
void bicubicIterations(w2ximg::Image3f &image, int iterations) {
    for (int i = 0; i < iterations; i++) image = w2ximg::resize(image, image.width * 2, image.height * 2, w2ximg::CUBIC);
}
double shrinkRatioOf(double scaleRatio, int iterTimesTwiceScaling) {   // :109-113, 0 = none
    if (static_cast<int>(scaleRatio) != std::pow(2, iterTimesTwiceScaling)) return scaleRatio / std::pow(2.0, static_cast<double>(iterTimesTwiceScaling));
    return 0.0;
}
void shrinkImage(w2ximg::Image3f &image, double shrinkRatio) {         // :158-167
    if (shrinkRatio == 0.0) return;
    int lw = static_cast<int>(static_cast<double>(image.width * shrinkRatio));
    int lh = static_cast<int>(static_cast<double>(image.height * shrinkRatio));
    image = w2ximg::resize(image, lw, lh, w2ximg::LINEAR);
}
std::vector<uint8_t> rgb8(w2ximg::Image3f &image) {                      // :171-172
    w2ximg::yuv2rgb(image);
    return w2ximg::to_u8(image);
}
std::string autoOutputName(const std::string &inputFile, const std::string &mode, int nrLevel, double scaleRatio) {   // :173-189
    std::string outputFileName = inputFile;
    size_t tailDot = outputFileName.find_last_of('.');
    if (tailDot != std::string::npos) outputFileName.erase(tailDot, outputFileName.length());
    outputFileName = outputFileName + "(" + mode + ")";
    if (mode.find("noise") != mode.npos) outputFileName = outputFileName + "(Level" + std::to_string(nrLevel) + ")";
    if (mode.find("scale") != mode.npos) outputFileName = outputFileName + "(x" + std::to_string(scaleRatio) + ")";
    return outputFileName + ".png";
}
bool writeImage(const std::string &outputFileName, const std::vector<uint8_t> &out8, int width, int height) {   // :190
    if (w2xio::imwrite(outputFileName, out8.data(), width, height)) return true;
    std::cerr << ("Error : couldn't write " + outputFileName + "\n") << std::flush;
    return false;
}

// ---- --input_list: many images in one process ----
// Threads that run queued tasks in queue order (-j of them); the destructor runs what is still queued, then joins.
class Workers {
public:
    explicit Workers(int n) {
        for (int i = 0; i < n; i++) threads_.emplace_back([this] { loop(); });
    }
    ~Workers() {
        {
            std::lock_guard<std::mutex> lock(mu_);
            stop_ = true;
        }
        cv_.notify_all();
        for (auto &t : threads_) t.join();
    }
    void run(std::function<void()> task) {
        {
            std::lock_guard<std::mutex> lock(mu_);
            queue_.push_back(std::move(task));
        }
        cv_.notify_one();
    }

private:
    void loop() {
        for (;;) {
            std::function<void()> task;
            {
                std::unique_lock<std::mutex> lock(mu_);
                cv_.wait(lock, [this] { return stop_ || !queue_.empty(); });
                if (queue_.empty()) return;
                task = std::move(queue_.front());
                queue_.pop_front();
            }
            task();
        }
    }
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<std::function<void()>> queue_;
    bool stop_ = false;
    std::vector<std::thread> threads_;
};

// A count of outstanding tasks that a thread can wait for.
class Pending {
public:
    void add(int n) {
        std::lock_guard<std::mutex> lock(mu_);
        left_ += n;
    }
    void done() {
        std::lock_guard<std::mutex> lock(mu_);
        if (--left_ == 0) cv_.notify_all();
    }
    void wait() {
        std::unique_lock<std::mutex> lock(mu_);
        cv_.wait(lock, [this] { return left_ == 0; });
    }

private:
    std::mutex mu_;
    std::condition_variable cv_;
    int left_ = 0;
};

[[noreturn]] void batchError(const std::string &text) {   // a check before any work: nothing was decoded, loaded or written
    std::cerr << "Error : " << text << std::endl;
    std::exit(1);
}

// --input_list <file>: every image of the list through the passes of a single-image run with the same flags, and byte for byte the
// PNG that run writes.  The list is cut, in input order, into groups whose Y planes go through ONE w2x_convert_planes_chain call (packed
// into shared frames; with several GPUs w2x_multi_convert_planes_chain); while group g is on the GPU, the workers decode group g + 1,
// run group g's bicubic U/V iterations and finish group g - 1 (merge, shrink, RGB, PNG).  Returns the exit code.
int runBatch(const CmdLine &cmd) {
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_start = now();
    const std::string mode = cmd.get("mode"), modelDir = cmd.get("model_dir"), listFile = cmd.get("input_list"), outDir = cmd.get("output_file");
    const int nrLevel = std::atoi(cmd.get("noise_level").c_str());
    const double scaleRatio = std::strtod(cmd.get("scale_ratio").c_str(), nullptr);
    const bool tta = cmd.get("tta") == "1";
    const bool noisePhase = mode == "noise" || mode == "noise_scale", scalePhase = mode == "scale" || mode == "noise_scale";
    const int iterTimesTwiceScaling = static_cast<int>(std::ceil(std::log2(scaleRatio)));
    const int upscales = scalePhase ? std::max(iterTimesTwiceScaling, 0) : 0;
    const double shrinkRatio = scalePhase ? shrinkRatioOf(scaleRatio, iterTimesTwiceScaling) : 0.0;

    // ---- checks before any work ----
    // A group's cost is the sum over its images of the Y plane's largest step output in pixels (x8 for a TTA chain); a group closes
    // before the image that would take it past the budget.  It bounds the host and device memory of a group, never the bits.
    uint64_t budget = uint64_t(1) << 25;
    if (const char *b = std::getenv("W2X_CLI_BATCH_PIXELS")) {
        char *end = nullptr;
        const unsigned long long v = std::strtoull(b, &end, 10);
        if (end == b || *end || v == 0 || *b == '-') batchError(std::string("W2X_CLI_BATCH_PIXELS must be a positive number of pixels (got \"") + b + "\")");
        budget = v;
    }
    const bool toDir = outDir != "(auto)";
    std::error_code ec;
    if (toDir && !std::filesystem::is_directory(outDir, ec)) batchError("-o " + outDir + " is not a directory");
    std::ifstream list(listFile);
    if (!list) batchError("couldn't open " + listFile);
    struct Item {
        std::string input, output;
        bool decoded = false, ok = false;
        uint64_t cost = 0;
        w2ximg::Image3f image;
        w2xc::Plane y, yout;
    };
    std::vector<Item> items;
    for (std::string line; std::getline(list, line);) {
        if (!line.empty() && line.back() == '\r') line.pop_back();
        if (line.empty()) continue;
        Item it;
        it.input = line;
        it.output = autoOutputName(line, mode, nrLevel, scaleRatio);
        if (toDir) it.output = outDir + (outDir.back() == '/' ? "" : "/") + it.output.substr(it.output.find_last_of('/') + 1);   // npos + 1 = 0
        items.push_back(std::move(it));
    }
    if (items.empty()) batchError(listFile + " names no input file");
    {
        std::map<std::string, size_t> seen;   // the same file however it is spelt (./a.png, a.png, a/../a.png, symbolic links)
        for (size_t i = 0; i < items.size(); i++) {
            std::filesystem::path p = std::filesystem::weakly_canonical(std::filesystem::absolute(items[i].output, ec), ec);
            auto r = seen.emplace(ec ? items[i].output : p.string(), i);
            if (!r.second)
                batchError(items[r.first->second].input + " and " + items[i].input + " would both be written to " + items[i].output);
        }
    }
    const size_t n = items.size();

    // ---- models, once for the run ----
    std::vector<std::unique_ptr<w2xc::Model>> noiseModels, scaleModels;
    const std::string noiseFile = modelDir + "/noise" + std::to_string(nrLevel) + "_model.json", scaleFile = modelDir + "/scale2.0x_model.json";
    const bool gpu = noisePhase || upscales > 0;   // an image with no GPU step only gets the host passes
    std::thread gpu_warmup;
    if (gpu) gpu_warmup = std::thread([] { w2xc::gpuRuntime::warmup(); });   // CUDA context creation overlaps model parsing and decoding
    auto leave = [&](int code) {
        if (gpu_warmup.joinable()) gpu_warmup.join();
        return code;
    };
    if (noisePhase) w2xc::modelUtility::prefetchModelFromJSON(noiseFile);
    if (scalePhase) w2xc::modelUtility::prefetchModelFromJSON(scaleFile);
    if (noisePhase && !w2xc::modelUtility::generateModelFromJSON(noiseFile, noiseModels)) return leave(-1);
    if (scalePhase && !w2xc::modelUtility::generateModelFromJSON(scaleFile, scaleModels)) return leave(-1);
    w2xc::modelUtility::getInstance().setNumberOfJobs(std::atoi(cmd.get("jobs").c_str()));
    const std::vector<w2xc::ChainStep> steps = chainSteps(noisePhase, upscales, tta, noiseModels, scaleModels);

    // ---- the pipeline ----
    struct Group {
        size_t begin = 0, end = 0;
        Pending decoded, coloured, finished;
    };
    std::vector<std::unique_ptr<Group>> groups;
    std::mutex print_mu;
    std::vector<char> state(n, 0);   // 0 = not finished, 1 = written, 2 = not written
    size_t next_line = 0;
    bool all_written = true;
    auto report = [&](size_t i, bool written) {   // "<input> -> <output>" once the file is closed, in input order
        std::lock_guard<std::mutex> lock(print_mu);
        state[i] = written ? 1 : 2;
        all_written = all_written && written;
        for (; next_line < n && state[next_line]; next_line++)
            if (state[next_line] == 1) std::cout << items[next_line].input << " -> " << items[next_line].output << std::endl;
    };
    auto decode = [&](Item &it) {
        w2xio::Image8 in8;
        it.decoded = true;
        if (!readImage(it.input, in8)) return;   // skipped: costs nothing, is not converted, and the run ends with -1
        it.ok = true;
        it.image = yuvImage(in8);
        it.cost = ((uint64_t)it.image.width * it.image.height << (2 * upscales)) * (tta ? 8 : 1);
        if (!gpu) return;
        it.y = plane_of(it.image, 0);
        it.yout.create(it.image.width << upscales, it.image.height << upscales);
    };
    auto finish = [&](Item &it, size_t i, Group &g) {
        bool written = false;
        if (it.ok) {
            if (gpu) w2ximg::set_channel(it.image, 0, it.yout.data, it.yout.stride_bytes / 4);   // merge, :98 and :154
            shrinkImage(it.image, shrinkRatio);
            const std::vector<uint8_t> out8 = rgb8(it.image);
            written = writeImage(it.output, out8, it.image.width, it.image.height);
        }
        it.image = w2ximg::Image3f();
        it.y = it.yout = w2xc::Plane();
        report(i, written);
        g.finished.done();
    };
    int code = 0;
    double t_conv = 0.0;
    {
        Workers workers(std::max(1, std::min(std::atoi(cmd.get("jobs").c_str()), 64)));
        auto startDecoding = [&](size_t begin) {   // one task, in input order: the first image that does not fit opens the next group
            groups.emplace_back(new Group);
            Group *g = groups.back().get();
            g->begin = begin;
            g->decoded.add(1);
            workers.run([&, g] {
                uint64_t cost = 0;
                size_t i = g->begin;
                for (; i < n; i++) {
                    if (!items[i].decoded) decode(items[i]);
                    if (i > g->begin && cost + items[i].cost > budget) break;
                    cost += items[i].cost;
                }
                g->end = i;
                g->decoded.done();
            });
        };
        startDecoding(0);
        for (size_t gi = 0; gi < groups.size(); gi++) {
            Group &g = *groups[gi];
            g.decoded.wait();
            if (gi >= 2) groups[gi - 2]->finished.wait();   // at most three groups on the host: finishing, converting, decoding
            if (g.end < n) startDecoding(g.end);
            std::vector<w2xc::Plane> in, out;
            std::vector<size_t> index;
            for (size_t i = g.begin; i < g.end; i++) {
                if (!items[i].ok) continue;
                index.push_back(i);
                in.push_back(items[i].y);
                out.push_back(items[i].yout);
                if (upscales > 0) {
                    g.coloured.add(1);
                    workers.run([&, i] { bicubicIterations(items[i].image, upscales); g.coloured.done(); });
                }
            }
            bool ok = true;
            if (gpu && !in.empty()) {
                if (gpu_warmup.joinable()) gpu_warmup.join();
                const double t0 = now();
                ok = w2xc::convertPlanesChainWithModels(in, out, steps);
                t_conv += now() - t0;
            }
            g.coloured.wait();
            if (!ok) {   // nothing of this group is written; the groups before it finish
                std::cerr << "w2xc::convertWithModels : something error has occured.\nstop." << std::endl;
                code = 1;
                break;
            }
            for (size_t k = 0; k < index.size(); k++) items[index[k]].yout = out[k];
            g.finished.add((int)(g.end - g.begin));
            for (size_t i = g.begin; i < g.end; i++) workers.run([&, i] { finish(items[i], i, g); });
        }
    }   // the workers finish what is queued
    if (code == 0 && !all_written) code = -1;
    if (std::getenv("W2X_CLI_TIMING"))
        std::cerr << "{\"w2x_cli_batch_timing_ms\": {\"images\": " << n << ", \"groups\": " << groups.size() << ", \"convert\": " << t_conv
                  << ", \"total\": " << now() - t_start << "}}" << std::endl;
    if (code == 0) std::cout << "process successfully done!" << std::endl;
    return leave(code);
}

}  // namespace

int main(int argc, char **argv) {
    CmdLine cmd;
    cmd.add("i", "input_file", "path to input image file (you should input full path)", true, "", "string").alternative = "input_list";
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
    // a file naming one input image per line, in place of -i: one process, the models loaded once, and the images' Y planes converted
    // in groups by one collection call each (runBatch); -o, if given, names the directory the (auto)-named outputs go to
    cmd.add("", "input_list", "file naming one input image per line", false, "", "string").hidden = true;
    cmd.parse(argc, argv);
    const bool tta = cmd.get("tta") == "1";
    const bool batch = cmd.isSet("input_list");
    if (!batch) {
        const int gpus = w2xc::gpuRuntime::plannedNumberOfGpus(std::atoi(cmd.get("gpus").c_str()));
        if (tta && gpus > 1) {   // a TTA step has no multi-GPU form (w2x_multi_convert_chain refuses it)
            std::cerr << "Error : --tta 1 runs on one GPU; it cannot be combined with " << gpus << " GPUs (--gpus / W2X_GPUS / W2X_DEVICES)." << std::endl;
            std::exit(1);
        }
    }
    if (std::atoi(cmd.get("gpus").c_str()) > 1) w2xc::gpuRuntime::setNumberOfGpus(std::atoi(cmd.get("gpus").c_str()));
    if (batch) {   // every file is written and closed: skip the teardown as below
        const int code = runBatch(cmd);
        std::cout.flush();
        std::cerr.flush();
        if (!std::getenv("W2X_CLI_FULL_TEARDOWN")) std::_Exit(code);
        return code;
    }
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
    w2xio::Image8 in8;
    if (!readImage(inputFile, in8)) leave(-1);
    const double t_read = now();
    w2ximg::Image3f image = yuvImage(in8);

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
        const int chainedIterations = chained ? iterTimesTwiceScaling : 0;
        const std::vector<w2xc::ChainStep> steps = chainSteps(noisePhase, chainedIterations, tta, noiseModels, scaleModels);
        w2xc::Plane imageY = plane_of(image, 0), out;
        wait_for_gpu();
        std::thread colour([&] { bicubicIterations(image, chainedIterations); });
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
        const double shrinkRatio = shrinkRatioOf(scaleRatio, iterTimesTwiceScaling);
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
        shrinkImage(image, shrinkRatio);
    }

    const std::vector<uint8_t> out8 = rgb8(image);
    std::string outputFileName = cmd.get("output_file");
    if (outputFileName == "(auto)") outputFileName = autoOutputName(inputFile, mode, nrLevel, scaleRatio);
    const double t_write0 = now();
    if (!writeImage(outputFileName, out8, image.width, image.height)) leave(-1);
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
