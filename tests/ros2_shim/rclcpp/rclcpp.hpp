// ROS 2 shim (test code only): the part of rclcpp that ros2/urf_ros2_node.cpp uses, with rclcpp's names and signatures,
// so that the node compiles and runs in tests/kat/ros2_glue_entry.cpp without a ROS 2 installation. Nothing leaves the
// process:
//   - a publisher keeps every message it is given (shim_sent), a subscription keeps its callback (shim_deliver);
//   - the log macros keep their level and text (shim_logs); the throttled ones log every call;
//   - Node takes NodeOptions().parameter_overrides(...), runs the on-set callbacks for declare_parameter, set_parameters
//     (one parameter per call) and set_parameters_atomically (all in one call), and stores the values they accept.
// Descriptors are recorded (shim_descriptors) but their ranges and read-only flags are not enforced, nor are undeclared
// names refused: the tests exercise the node's own checks.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <functional>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include <rcl_interfaces/msg/parameter_descriptor.hpp>
#include <rcl_interfaces/msg/set_parameters_result.hpp>

namespace rclcpp {

enum ParameterType : uint8_t {
  PARAMETER_NOT_SET = 0, PARAMETER_BOOL = 1, PARAMETER_INTEGER = 2, PARAMETER_DOUBLE = 3, PARAMETER_STRING = 4,
};

inline std::string to_string(ParameterType t) {
  switch (t) {
    case PARAMETER_BOOL: return "bool";
    case PARAMETER_INTEGER: return "integer";
    case PARAMETER_DOUBLE: return "double";
    case PARAMETER_STRING: return "string";
    default: return "not set";
  }
}

class ParameterValue {
 public:
  ParameterValue() = default;
  explicit ParameterValue(bool v) : type_(PARAMETER_BOOL), b_(v) {}
  explicit ParameterValue(int v) : type_(PARAMETER_INTEGER), i_(v) {}
  explicit ParameterValue(int64_t v) : type_(PARAMETER_INTEGER), i_(v) {}
  explicit ParameterValue(double v) : type_(PARAMETER_DOUBLE), d_(v) {}
  explicit ParameterValue(const std::string& v) : type_(PARAMETER_STRING), s_(v) {}
  explicit ParameterValue(const char* v) : type_(PARAMETER_STRING), s_(v) {}
  ParameterType get_type() const { return type_; }
  bool as_bool() const { want(PARAMETER_BOOL); return b_; }
  int64_t as_int() const { want(PARAMETER_INTEGER); return i_; }
  double as_double() const { want(PARAMETER_DOUBLE); return d_; }
  const std::string& as_string() const { want(PARAMETER_STRING); return s_; }

 private:
  void want(ParameterType t) const {
    if (t != type_) throw std::runtime_error("wrong parameter type, expected " + to_string(t) + " got " + to_string(type_));
  }
  ParameterType type_ = PARAMETER_NOT_SET;
  bool b_ = false;
  int64_t i_ = 0;
  double d_ = 0.0;
  std::string s_;
};

class Parameter {
 public:
  Parameter() = default;
  Parameter(const std::string& name, const ParameterValue& value) : name_(name), value_(value) {}
  template <typename T>
  Parameter(const std::string& name, T value) : Parameter(name, ParameterValue(value)) {}
  const std::string& get_name() const { return name_; }
  ParameterType get_type() const { return value_.get_type(); }
  std::string get_type_name() const { return to_string(get_type()); }
  const ParameterValue& get_parameter_value() const { return value_; }
  bool as_bool() const { return value_.as_bool(); }
  int64_t as_int() const { return value_.as_int(); }
  double as_double() const { return value_.as_double(); }
  const std::string& as_string() const { return value_.as_string(); }

 private:
  std::string name_;
  ParameterValue value_;
};

namespace exceptions {
struct InvalidParameterValueException : std::runtime_error {
  using std::runtime_error::runtime_error;
};
}  // namespace exceptions

class NodeOptions {
 public:
  NodeOptions& parameter_overrides(const std::vector<Parameter>& p) { overrides_ = p; return *this; }
  const std::vector<Parameter>& parameter_overrides() const { return overrides_; }

 private:
  std::vector<Parameter> overrides_;
};

enum class ReliabilityPolicy { BestEffort, Reliable, SystemDefault };
struct KeepLast {
  explicit KeepLast(size_t depth) : depth(depth) {}
  size_t depth;
};
class QoS {
 public:
  QoS(const KeepLast& k) : depth_(k.depth) {}  // NOLINT: implicit, as in rclcpp
  explicit QoS(size_t depth) : depth_(depth) {}
  QoS& best_effort() { rel_ = ReliabilityPolicy::BestEffort; return *this; }
  QoS& reliable() { rel_ = ReliabilityPolicy::Reliable; return *this; }
  ReliabilityPolicy reliability() const { return rel_; }
  size_t depth() const { return depth_; }

 private:
  size_t depth_;
  ReliabilityPolicy rel_ = ReliabilityPolicy::Reliable;
};

struct Time {
  int64_t nanoseconds() const { return 0; }
};
struct Clock {
  using SharedPtr = std::shared_ptr<Clock>;
  Time now() const { return Time(); }
};

class Logger {
 public:
  explicit Logger(std::string name) : name_(std::move(name)) {}
  const char* get_name() const { return name_.c_str(); }

 private:
  std::string name_;
};

struct ShimLog {
  char level;           // 'I', 'W', 'E', 'F'
  std::string text;
};
inline std::vector<ShimLog>& shim_logs() { static std::vector<ShimLog> l; return l; }
inline void shim_log(const Logger&, char level, const char* fmt, ...) __attribute__((format(printf, 3, 4)));
inline void shim_log(const Logger&, char level, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  std::vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  shim_logs().push_back({level, buf});
}

struct PublisherBase {
  virtual ~PublisherBase() = default;
};
template <typename MessageT>
class Publisher : public PublisherBase {
 public:
  using SharedPtr = std::shared_ptr<Publisher>;
  Publisher(std::string topic, const QoS& qos) : topic_(std::move(topic)), qos_(qos) {}
  void publish(std::unique_ptr<MessageT> msg) { shim_sent.push_back(std::move(msg)); }
  void publish(const MessageT& msg) { shim_sent.push_back(std::make_unique<MessageT>(msg)); }
  const char* get_topic_name() const { return topic_.c_str(); }
  const QoS& shim_qos() const { return qos_; }
  std::vector<std::unique_ptr<MessageT>> shim_sent;

 private:
  std::string topic_;
  QoS qos_;
};

struct SubscriptionBase {
  virtual ~SubscriptionBase() = default;
};
template <typename MessageT>
class Subscription : public SubscriptionBase {
 public:
  using SharedPtr = std::shared_ptr<Subscription>;
  Subscription(std::string topic, const QoS& qos, std::function<void(std::shared_ptr<const MessageT>)> cb)
      : topic_(std::move(topic)), qos_(qos), cb_(std::move(cb)) {}
  const char* get_topic_name() const { return topic_.c_str(); }
  const QoS& shim_qos() const { return qos_; }
  void shim_deliver(std::shared_ptr<const MessageT> msg) { cb_(std::move(msg)); }

 private:
  std::string topic_;
  QoS qos_;
  std::function<void(std::shared_ptr<const MessageT>)> cb_;
};

namespace node_interfaces {
struct OnSetParametersCallbackHandle {
  using SharedPtr = std::shared_ptr<OnSetParametersCallbackHandle>;
  using OnSetParametersCallbackType = std::function<rcl_interfaces::msg::SetParametersResult(const std::vector<Parameter>&)>;
  OnSetParametersCallbackType callback;
};
}  // namespace node_interfaces

class Node : public std::enable_shared_from_this<Node> {
 public:
  using SharedPtr = std::shared_ptr<Node>;
  using OnSetParametersCallbackHandle = node_interfaces::OnSetParametersCallbackHandle;

  explicit Node(const std::string& node_name, const NodeOptions& options = NodeOptions())
      : name_(node_name), options_(options), logger_(node_name), clock_(std::make_shared<Clock>()) {}
  virtual ~Node() = default;

  const char* get_name() const { return name_.c_str(); }
  Logger get_logger() const { return logger_; }
  Clock::SharedPtr get_clock() { return clock_; }

  const ParameterValue& declare_parameter(const std::string& name, const ParameterValue& default_value,
                                          const rcl_interfaces::msg::ParameterDescriptor& descriptor =
                                              rcl_interfaces::msg::ParameterDescriptor(),
                                          bool ignore_override = false) {
    if (values_.count(name)) throw std::runtime_error("parameter '" + name + "' has already been declared");
    Parameter p(name, default_value);
    if (!ignore_override)
      for (const Parameter& o : options_.parameter_overrides()) if (o.get_name() == name) p = o;
    const rcl_interfaces::msg::SetParametersResult r = run_callbacks({p});
    if (!r.successful) throw exceptions::InvalidParameterValueException("parameter '" + name + "' could not be set: " + r.reason);
    shim_descriptors[name] = descriptor;
    return values_[name] = p.get_parameter_value();
  }
  Parameter get_parameter(const std::string& name) const {
    auto it = values_.find(name);
    if (it == values_.end()) throw std::runtime_error("parameter '" + name + "' is not declared");
    return Parameter(name, it->second);
  }

  OnSetParametersCallbackHandle::SharedPtr add_on_set_parameters_callback(OnSetParametersCallbackHandle::OnSetParametersCallbackType cb) {
    auto h = std::make_shared<OnSetParametersCallbackHandle>();
    h->callback = std::move(cb);
    callbacks_.push_back(h);
    return h;
  }
  std::vector<rcl_interfaces::msg::SetParametersResult> set_parameters(const std::vector<Parameter>& params) {
    std::vector<rcl_interfaces::msg::SetParametersResult> out;
    for (const Parameter& p : params) out.push_back(set_parameters_atomically({p}));
    return out;
  }
  rcl_interfaces::msg::SetParametersResult set_parameters_atomically(const std::vector<Parameter>& params) {
    const rcl_interfaces::msg::SetParametersResult r = run_callbacks(params);
    if (r.successful) for (const Parameter& p : params) values_[p.get_name()] = p.get_parameter_value();
    return r;
  }

  template <typename MessageT>
  typename Publisher<MessageT>::SharedPtr create_publisher(const std::string& topic, const QoS& qos) {
    auto p = std::make_shared<Publisher<MessageT>>(topic, qos);
    shim_publishers[topic] = p;
    return p;
  }
  template <typename MessageT, typename CallbackT>
  typename Subscription<MessageT>::SharedPtr create_subscription(const std::string& topic, const QoS& qos, CallbackT&& cb) {
    auto s = std::make_shared<Subscription<MessageT>>(topic, qos, std::function<void(std::shared_ptr<const MessageT>)>(std::forward<CallbackT>(cb)));
    shim_subscriptions[topic] = s;
    return s;
  }

  // shim only: what the node created and declared, by topic and by parameter name
  std::map<std::string, std::shared_ptr<PublisherBase>> shim_publishers;
  std::map<std::string, std::shared_ptr<SubscriptionBase>> shim_subscriptions;
  std::map<std::string, rcl_interfaces::msg::ParameterDescriptor> shim_descriptors;
  size_t shim_callback_count() const { return callbacks_.size(); }

 private:
  rcl_interfaces::msg::SetParametersResult run_callbacks(const std::vector<Parameter>& params) {
    rcl_interfaces::msg::SetParametersResult r;
    r.successful = true;
    for (const auto& h : callbacks_) {
      r = h->callback(params);
      if (!r.successful) break;
    }
    return r;
  }

  std::string name_;
  NodeOptions options_;
  Logger logger_;
  Clock::SharedPtr clock_;
  std::map<std::string, ParameterValue> values_;
  std::vector<OnSetParametersCallbackHandle::SharedPtr> callbacks_;
};

}  // namespace rclcpp

#define RCLCPP_INFO(logger, ...) ::rclcpp::shim_log(logger, 'I', __VA_ARGS__)
#define RCLCPP_WARN(logger, ...) ::rclcpp::shim_log(logger, 'W', __VA_ARGS__)
#define RCLCPP_ERROR(logger, ...) ::rclcpp::shim_log(logger, 'E', __VA_ARGS__)
#define RCLCPP_FATAL(logger, ...) ::rclcpp::shim_log(logger, 'F', __VA_ARGS__)
// rclcpp takes a Clock& and a duration in milliseconds; both are only type-checked here
#define RCLCPP_ERROR_THROTTLE(logger, clock, duration, ...) \
  do { (void)(clock).now(); (void)(duration); ::rclcpp::shim_log(logger, 'E', __VA_ARGS__); } while (0)
